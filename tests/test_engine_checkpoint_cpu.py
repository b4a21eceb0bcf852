"""BnetDDP's layout-free optimizer state (full_optimizer_state_dict / load_full_optimizer_state_dict) on the CPU: the shard
<-> full mapping at world sizes 1-8 against the flat buffer plan_buckets lays out, the round trip through another bucket
layout, torch.optim.SGD / AdamW taking the state over and handing it back, and every state the loader refuses.  Other world
sizes of the engine itself run on the GPU (tests/test_checkpoint_reshard.py)."""
import copy

import pytest
import torch
from engine_fakes import FakeComm, cpu_engine  # noqa: F401 - cpu_engine is a fixture
from engine_fakes import HYPER, batch, close_params, small_model, torch_step

from bagua_net_b200.parallel.ddp import (BnetDDP, full_from_shard, memory_flat, no_weight_decay_groups, plan_buckets,
                                         shard_from_full, shard_pieces)


# ------------------------------------------------------------------ the shard <-> full mapping
NUMELS = [1, 7, 8, 9, 3 * 5 * 7 * 2, 1000, 17, 8 * 3 * 3 * 3, 5, 4096 + 3, 3]    # (index 7: a channels_last filter)


def _flats(seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(n, generator=g) for n in NUMELS]


def _layout(es, world, bucket_mb):
    plan, total = plan_buckets(NUMELS, es, world, bucket_mb)
    return plan, total, [shard_pieces(plan, NUMELS, world, r) for r in range(world)]


def _shards(flats, plan, pieces, world):
    return [[shard_from_full(flats, pieces[r][k], torch.full((numel // world,), float("nan")))
             for k, (_, numel, _) in enumerate(plan)] for r in range(world)]


def _gather(shards, pieces):
    out = [torch.full((n,), float("nan")) for n in NUMELS]
    for r, per_bucket in enumerate(shards):
        for k, s in enumerate(per_bucket):
            full_from_shard(out, pieces[r][k], s)
    return out


@pytest.mark.parametrize("es", [2, 4], ids=["bf16", "fp32"])
@pytest.mark.parametrize("buckets", [(0.002, 1.0), (0.01, 0.0005), (1.0, 0.004)], ids=lambda b: f"{b[0]}-{b[1]}MB")
def test_shard_mapping_reshards_bitwise(es, buckets):
    """A random full state scattered to the shards of (W1, B1) is the flat buffer's shard, padding zero; gathered back and
    scattered again through (W2, B2) and gathered, it is bitwise the state it started as, for every W1, W2 in 1..8."""
    full = _flats(1)
    seen = {"straddle": 0, "empty": 0}
    for w1 in range(1, 9):
        plan, total, pieces = _layout(es, w1, buckets[0])
        shards = _shards(full, plan, pieces, w1)
        flat = torch.zeros(total)                          # the oracle: the flat buffer of plan_buckets, sliced per rank
        for start, numel, members in plan:
            for pi, off in members:
                flat[off:off + NUMELS[pi]] = full[pi]
        for start, numel, _ in plan:
            shard = numel // w1
            for r in range(w1):
                k = [s for s, _, _ in plan].index(start)
                assert torch.equal(shards[r][k], flat[start + r * shard:start + (r + 1) * shard])
                seen["empty"] += not pieces[r][k]
        for pi in range(len(NUMELS)):
            owners = {r for r in range(w1) for ps in pieces[r] for q, *_ in ps if q == pi}
            seen["straddle"] += len(owners) > 1
            covered = sorted((p0, n) for r in range(w1) for ps in pieces[r] for q, p0, n, _ in ps if q == pi)
            assert sum(n for _, n in covered) == NUMELS[pi] and all(a + n == b for (a, n), (b, _) in zip(covered, covered[1:]))
        back = _gather(shards, pieces)
        for w2 in range(1, 9):
            plan2, _, pieces2 = _layout(es, w2, buckets[1])
            again = _gather(_shards(back, plan2, pieces2, w2), pieces2)
            assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(again, full)), (w1, w2)
    assert seen["straddle"] and (seen["empty"] or buckets[0] == 1.0)


def test_memory_flat_follows_the_flat_buffer_layout(cpu_engine):
    """A channels_last filter is NHWC in the flat buffer: memory_flat of the engine's parameter is that slice of the buffer,
    and memory_flat of a channels_last copy lists its elements in the same order."""
    net = small_model(channels_last=True)
    eng = BnetDDP(net, comm=FakeComm(), bucket_mb=0.002)
    w = net[0].weight
    assert not w.is_contiguous() and w.is_contiguous(memory_format=torch.channels_last)
    v = memory_flat(w)
    assert v.data_ptr() == w.data_ptr() and v.numel() == w.numel()
    off = (w.data_ptr() - eng.flat_param.data_ptr()) // 4
    assert torch.equal(v, eng.flat_param[off:off + w.numel()])
    c = torch.empty_like(w).copy_(w)
    assert torch.equal(memory_flat(c), v) and torch.equal(memory_flat(w.contiguous()), w.reshape(-1))


# ------------------------------------------------------------------ the engine's full state
def _groups(net):
    """Biases without decay, the head's weight at 4x the lr, the rest the default group: torch numbering != module order."""
    return [{"params": no_weight_decay_groups(net)[0]["params"], "weight_decay": 0.0},
            {"params": [net[-1].weight], "lr_scale": 4.0}]


CASES = {"sgd": dict(optimizer="sgd", **HYPER["sgd"]),
         "adamw-ema-groups": dict(optimizer="adamw", **HYPER["adamw"], ema_decay=0.5, groups=True),
         "lars-clip-accum": dict(optimizer="lars", **HYPER["lars"], max_grad_norm=0.5, accumulation_steps=2)}


def _engine(case, bucket_mb):
    kw = dict(CASES[case])
    groups = kw.pop("groups", False)
    net = small_model()
    return net, BnetDDP(net, comm=FakeComm(), bucket_mb=bucket_mb, param_groups=_groups(net) if groups else None, **kw)


def assert_same(a, b, path="state"):
    """Equal dicts, lists and numbers; tensors of the same dtype, shape, strides and bits."""
    assert type(a) is type(b), path
    if isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and a.shape == b.shape and a.stride() == b.stride(), path
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), path
    elif isinstance(a, dict):
        assert list(a) == list(b), path
        for k in a:
            assert_same(a[k], b[k], f"{path}[{k!r}]")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, f"{path}[{i}]")
    else:
        assert a == b, path


def _padding_is_zero(eng):
    numels = [p.numel() for p in eng._params]
    for b, pieces in zip(eng.buckets, shard_pieces(eng._plan, numels, 1, 0)):
        pad = torch.ones(b.master.numel(), dtype=torch.bool)
        for _, _, n, s0 in pieces:
            pad[s0:s0 + n] = False
        for t in b.state + ((b.ema,) if b.ema is not None else ()):
            assert bool((t[pad] == 0).all())


@pytest.mark.parametrize("case", CASES)
def test_full_state_round_trip_through_another_bucket_layout(cpu_engine, case):
    net, eng = _engine(case, 0.002)
    k = eng.accumulation_steps
    for step in range(3):
        eng.train_step(*batch(step, 4 * k, 300))
        if step == 1 and eng.param_groups:
            eng.set_param_group(0, lr_scale=0.5)
    full = copy.deepcopy(eng.full_optimizer_state_dict())
    assert set(full) == {"state", "param_groups", "bnet"} and len(full["state"]) == len(eng._params)
    filters = 0
    for i, j in enumerate(eng._torch_order()):
        for t in [full["bnet"]["master"][i]] + [t for t in full["state"][i].values() if t.dim()]:
            assert t.dtype == torch.float32 and t.shape == eng._params[j].shape and t.stride() == eng._params[j].stride()
            filters += t.dim() == 4 and not t.is_contiguous() and t.is_contiguous(memory_format=torch.channels_last)
    assert filters                                          # (channels_last filters stay channels_last)
    net2, other = _engine(case, 0.0005)
    assert len(other.buckets) > len(eng.buckets)
    for b in other.buckets:                                 # (what the load must overwrite, padding included)
        for t in b.state + ((b.ema,) if b.ema is not None else ()):
            t.fill_(7.0)
    net2.load_state_dict(net.state_dict())
    other.load_full_optimizer_state_dict(copy.deepcopy(full))
    _padding_is_zero(other)
    assert_same(other.full_optimizer_state_dict(), full)
    if eng.param_groups is not None:
        assert [(g["lr"], g["lr_scale"], g["weight_decay"], len(g["params"])) for g in other.param_groups] == \
            [(g["lr"], g["lr_scale"], g["weight_decay"], len(g["params"])) for g in eng.param_groups]
    x, y = batch(9, 4 * k, 300)
    eng.train_step(x, y)
    other.train_step(x, y)
    close_params(net2, net, 1e-6, case, rtol=1e-6)


# ------------------------------------------------------------------ torch.optim interop
def _torch_opt(optimizer, ref, eng, net):
    """torch.optim built from `eng.param_groups` (or one group) on `ref`'s matching parameters."""
    index = {id(p): i for i, p in enumerate(net.parameters())}
    rp = list(ref.parameters())
    groups = eng.param_groups or [{"params": list(net.parameters()), "lr": eng.lr, "weight_decay": eng.weight_decay}]
    groups = [{"params": [rp[index[id(p)]] for p in g["params"]], "lr": g["lr"], "weight_decay": g["weight_decay"]}
              for g in groups]
    if optimizer == "adamw":
        return torch.optim.AdamW(groups, betas=HYPER["adamw"]["betas"], eps=HYPER["adamw"]["eps"])
    return torch.optim.SGD(groups, momentum=HYPER["sgd"]["momentum"])


@pytest.mark.parametrize("groups", [False, True], ids=["one-group", "groups"])
@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_engine_state_continues_in_torch_optim(cpu_engine, optimizer, groups):
    net = small_model()
    eng = BnetDDP(net, optimizer=optimizer, bucket_mb=0.002, comm=FakeComm(), param_groups=_groups(net) if groups else None,
                  **HYPER[optimizer])
    for step in range(3):
        eng.train_step(*batch(step, 8, 400))
    full = copy.deepcopy(eng.full_optimizer_state_dict())
    ref = small_model().double()
    ref.load_state_dict({n: t.double() for n, t in net.state_dict().items()})
    opt = _torch_opt(optimizer, ref, eng, net)
    opt.load_state_dict(full)
    for step in range(3, 6):
        x, y = batch(step, 8, 400)
        eng.train_step(x, y)
        torch_step(ref, opt, x, y)
    close_params(net, ref, 1e-5, (optimizer, groups), rtol=1e-4)


@pytest.mark.parametrize("groups", [False, True], ids=["one-group", "groups"])
@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_torch_optim_state_continues_in_engine(cpu_engine, optimizer, groups):
    net = small_model()
    eng = BnetDDP(net, optimizer=optimizer, bucket_mb=0.002, comm=FakeComm(), param_groups=_groups(net) if groups else None,
                  **HYPER[optimizer])
    ref = small_model().double()
    opt = _torch_opt(optimizer, ref, eng, net)
    for step in range(3):
        torch_step(ref, opt, *batch(step, 8, 500))
    if groups:                                    # the engine's lr is the last group's; the others become lr_scales
        for g, lr in zip(opt.param_groups, (0.7, 1.3, 0.5)):
            g["lr"] = lr * HYPER[optimizer]["lr"]
    with torch.no_grad():
        for p, q in zip(net.parameters(), ref.parameters()):
            p.copy_(q)
    eng.load_full_optimizer_state_dict(copy.deepcopy(opt.state_dict()))
    if groups:
        assert [g["lr_scale"] for g in eng.param_groups] == pytest.approx([1.4, 2.6, 1.0])
        assert eng.lr == pytest.approx(0.5 * HYPER[optimizer]["lr"])
    for step in range(3, 6):
        x, y = batch(step, 8, 500)
        eng.train_step(x, y)
        torch_step(ref, opt, x, y)
    close_params(net, ref, 1e-5, (optimizer, groups), rtol=1e-4)


def test_missing_torch_state_is_zero_state(cpu_engine):
    """A parameter without a state entry, or with momentum_buffer None (torch.optim.SGD at momentum 0), starts at zero."""
    net = small_model()
    eng = BnetDDP(net, bucket_mb=0.002, comm=FakeComm(), **HYPER["sgd"])
    ref = small_model().double()
    opt = _torch_opt("sgd", ref, eng, net)
    torch_step(ref, opt, *batch(0, 8, 600))
    sd = copy.deepcopy(opt.state_dict())
    del sd["state"][1]
    sd["state"][2]["momentum_buffer"] = None
    eng.load_full_optimizer_state_dict(sd)
    got = eng.full_optimizer_state_dict()["state"]
    assert not got[1]["momentum_buffer"].any() and not got[2]["momentum_buffer"].any()
    assert torch.equal(got[0]["momentum_buffer"], sd["state"][0]["momentum_buffer"].float())


# ------------------------------------------------------------------ what the loader refuses
def _torch_state(optimizer, eng, net, **kw):
    ref = small_model().double()
    opt = _torch_opt(optimizer, ref, eng, net)
    for g in opt.param_groups:
        g.update(kw)
    torch_step(ref, opt, *batch(0, 8, 700))
    return opt.state_dict()


def _set(sd, key, value, group=0):
    sd = copy.deepcopy(sd)
    sd["param_groups"][group][key] = value
    return sd


def test_load_rejects_what_the_engine_cannot_represent(cpu_engine):
    net = small_model()
    sgd = BnetDDP(net, bucket_mb=0.002, comm=FakeComm(), param_groups=_groups(net), **HYPER["sgd"])
    anet = small_model()
    adamw = BnetDDP(anet, optimizer="adamw", bucket_mb=0.002, comm=FakeComm(), param_groups=_groups(anet), **HYPER["adamw"])
    pnet = small_model()
    plain = BnetDDP(pnet, bucket_mb=0.002, comm=FakeComm(), **HYPER["sgd"])
    lnet = small_model()
    lars = BnetDDP(lnet, optimizer="lars", bucket_mb=0.002, comm=FakeComm(), **HYPER["lars"])
    s, a = _torch_state("sgd", sgd, net), _torch_state("adamw", adamw, anet)
    steps = copy.deepcopy(a)
    steps["state"][0]["step"] = torch.tensor(7.0)
    moved = copy.deepcopy(s)
    moved["param_groups"][0]["params"].append(moved["param_groups"][1]["params"].pop())
    shape = copy.deepcopy(s)
    shape["state"][0]["momentum_buffer"] = torch.zeros(3)
    rms = torch.optim.RMSprop(small_model().parameters(), momentum=0.9).state_dict()
    adam = torch.optim.Adam(small_model().parameters()).state_dict()
    one = torch.optim.SGD(small_model().parameters(), lr=0.1, momentum=0.9).state_dict()
    full_groups = sgd.full_optimizer_state_dict()
    full_plain = plain.full_optimizer_state_dict()
    ema_net = small_model()
    ema_full = BnetDDP(ema_net, bucket_mb=0.002, comm=FakeComm(), ema_decay=0.9, **HYPER["sgd"]).full_optimizer_state_dict()
    cases = [
        (sgd, _set(s, "momentum", 0.5), "differ in momentum"),
        (adamw, _set(a, "betas", (0.8, 0.99), 2), "differ in betas"),
        (adamw, _set(a, "eps", 1e-6, 1), "differ in eps"),
        (sgd, _set(s, "nesterov", True), "nesterov"),
        (sgd, _set(s, "dampening", 0.1, 2), "dampening"),
        (adamw, _set(a, "amsgrad", True), "amsgrad"),
        (sgd, _set(s, "maximize", True, 1), "maximize"),
        (adamw, _set(a, "maximize", True), "maximize"),
        (adamw, steps, "different AdamW steps"),
        (sgd, rms, "not a torch.optim.SGD or AdamW"),
        (adamw, adam, "not a torch.optim.SGD or AdamW"),
        (adamw, s, "cannot be loaded"),
        (lars, one, "cannot be loaded"),
        (sgd, a, "cannot be loaded"),
        (sgd, moved, "other parameters"),
        (sgd, shape, "shape"),
        (plain, s, "param groups and this engine none"),
        (sgd, one, "other parameters"),
        (plain, full_groups, "disagree on param groups"),
        (sgd, full_plain, "disagree on param groups"),
        (sgd, _set(s, "lr", 0.0, 2), "last param group has lr 0"),
        (plain, ema_full, "EMA"),
        (adamw, full_plain, "cannot be loaded"),
    ]
    before = {id(e): copy.deepcopy(e.full_optimizer_state_dict()) for e in (sgd, adamw, plain, lars)}
    for eng, state, msg in cases:
        with pytest.raises(ValueError, match=msg):
            eng.load_full_optimizer_state_dict(copy.deepcopy(state))
    for eng in (sgd, adamw, plain, lars):                   # a refused state changes nothing
        assert_same(eng.full_optimizer_state_dict(), before[id(eng)])
    sgd.load_full_optimizer_state_dict(_set(s, "lr", 0.0, 0))   # (lr 0 in another group is a scale of 0)
    assert sgd.param_groups[0]["lr_scale"] == 0.0
    zero = s
    for g in range(3):
        zero = _set(zero, "lr", 0.0, g)
    sgd.load_full_optimizer_state_dict(zero)                    # (every lr 0: scales 1)
    assert sgd.lr == 0.0 and [g["lr_scale"] for g in sgd.param_groups] == [1.0] * 3


@pytest.mark.parametrize("call", ["save", "load"])
def test_full_state_calls_refuse_mid_accumulation_and_inside_ema(cpu_engine, call):
    net = small_model()
    eng = BnetDDP(net, bucket_mb=0.002, comm=FakeComm(), accumulation_steps=2, ema_decay=0.5, **HYPER["sgd"])
    full = eng.full_optimizer_state_dict()
    run = eng.full_optimizer_state_dict if call == "save" else lambda: eng.load_full_optimizer_state_dict(full)
    x, y = batch(0, 2, 800)
    torch.nn.functional.cross_entropy(net(x), y).backward()
    eng.finish_step()
    with pytest.raises(ValueError, match="accumulation step"):
        run()
    torch.nn.functional.cross_entropy(net(x), y).backward()
    eng.finish_step()
    run()
    with eng.ema_parameters():
        with pytest.raises(ValueError, match="ema_parameters"):
            run()

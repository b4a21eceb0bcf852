"""BnetDDP(optimizer="lars")'s HOST logic on the CPU: the segment tables (a pure function, at world 1, 2, 3 and 8), the
staged step's launch order, the update against a float64 LARC + torch.optim.SGD reference (with and without clipping,
with accumulation, both memory formats, adopted and accumulated gradients), set_lr mid-run, the state dict, a bucket
without gradient and every rejected argument.  FakeComm does the stages in plain PyTorch with the kernels'
arithmetic; the kernels are covered on the GPU by tests/test_fused_lars.py."""
import copy
import math

import pytest
import torch
from engine_fakes import FakeComm, cpu_engine  # noqa: F401 - cpu_engine is a fixture
from engine_fakes import LARC, Branchy, batch, close_params, make_pair, torch_step
from engine_fakes import small_model as _model

from bagua_net_b200.parallel.comm import LARS_CHUNK, check_lars_segments, check_lars_tensors
from bagua_net_b200.parallel.ddp import BnetDDP, lars_segments, plan_buckets


# ------------------------------------------------------------------ the segment tables
def _tables(numels, es, world, bucket_mb):
    plan, _ = plan_buckets(numels, es, world, bucket_mb)
    return plan, {(k, r): lars_segments(m, numels, s, n, es, world, r) for k, (s, n, m) in enumerate(plan) for r in range(world)}


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("es", [2, 4])
def test_segment_tables_cover_every_shard_and_every_element_once(world, es):
    # odd sizes: a 1-element bias, tensors of one vector and less, one tensor wider than a shard, 2 chunks and a tail
    numels = [1, 7, 8, 9, 64 * 3 * 3 * 3, 5, 1000, 2 * LARS_CHUNK * 8 + 3, 17, 4096, 3]
    per_vec = 16 // es
    plan, tables = _tables(numels, es, world, 0.05)
    assert len(plan) >= 2
    for k, (start, numel, members) in enumerate(plan):
        shard = numel // world // per_vec
        owner = {}                                   # element of the flat buffer -> tensor of the segment holding it
        for r in range(world):
            t = tables[(k, r)]
            nslots = check_lars_segments(t, shard, len(numels))
            assert nslots == sum((n + LARS_CHUNK - 1) // LARS_CHUNK for _, n, _, _ in t)
            assert len({pi for _, _, pi, _ in t}) == len(t), "a tensor with two segments on one rank"
            for vec0, nvec, pi, _ in t:
                lo = start + (r * shard + vec0) * per_vec
                for x in range(lo, lo + nvec * per_vec):
                    assert x not in owner
                    owner[x] = pi
        assert sorted(owner) == list(range(start, start + numel))            # every element exactly once
        for pi, off in members:                                              # ... and a tensor's own in its segments
            assert all(owner[x] == pi for x in range(off, off + numels[pi]))
    if world > 1:                                                            # some tensor straddles a shard boundary
        straddle = [pi for (k, r), t in tables.items() for _, _, pi, _ in t
                    if any(pi == q for rr in range(world) if rr != r for _, _, q, _ in tables[(k, rr)])]
        assert straddle


def test_padding_only_shard_and_rejected_tables():
    # world 8, bf16: a bucket of 64 * 8 elements holding 9 -> shards 2..7 are padding only, owned by the last tensor
    t = [lars_segments([(0, 0)], [9], 0, 64 * 8, 2, 8, r) for r in range(8)]
    assert t[0] == [[0, 8, 0, 0]] and t[1] == [[0, 8, 0, 0]] and t[7] == [[0, 8, 0, 0]]
    good = [[0, 3, 0, 0], [3, LARS_CHUNK + 1, 1, 1], [LARS_CHUNK + 4, 4, 2, 3]]
    assert check_lars_segments(good, LARS_CHUNK + 8, 3) == 4
    bad = [
        [],                                                        # empty
        [[0, 3, 0, 0], [3, LARS_CHUNK + 1, 1, 1]],                 # does not reach the shard's end
        [[1, 2, 0, 0], [3, LARS_CHUNK + 5, 1, 1]],                 # does not start at 0
        [[0, 3, 0, 0], [2, LARS_CHUNK + 6, 1, 1]],                 # overlap
        [[0, 3, 0, 0], [4, LARS_CHUNK + 4, 1, 1]],                 # gap
        [[0, 3, 0, 0], [3, 0, 1, 1], [3, LARS_CHUNK + 5, 2, 1]],   # empty segment
        [[0, 3, 0, 0], [3, LARS_CHUNK + 5, 3, 1]],                 # tensor out of range
        [[0, 3, -1, 0], [3, LARS_CHUNK + 5, 1, 1]],                # negative tensor
        [[0, 3, 0, 0], [3, LARS_CHUNK + 5, 1, 2]],                 # wrong slot0
        [[0, LARS_CHUNK + 16, 0, 0]],                              # past the shard
    ]
    for b in bad:
        with pytest.raises(ValueError):
            check_lars_segments(b, LARS_CHUNK + 8, 3)
    check_lars_tensors([[0, 2, 0, 0], [2, 0, 1, 0]], 2)
    for b in ([[0, 3, 0, 0]], [[-1, 1, 0, 0]], [[1, -1, 0, 0]], []):
        with pytest.raises(ValueError):
            check_lars_tensors(b, 2)


# ------------------------------------------------------------------ the engine against float64 LARC + SGD
BATCH = 8


@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("clipped", [False, True], ids=["unclipped", "clipped"])
@pytest.mark.parametrize("direct_grads", ["1", "0"], ids=["adopted", "accumulated"])
@pytest.mark.parametrize("channels_last", [True, False])
def test_lars_engine_trains_like_larc_and_sgd(cpu_engine, k, clipped, direct_grads, channels_last):
    cpu_engine.setenv("BNET_DIRECT_GRADS", direct_grads)
    thr = 0.05 if clipped else None
    ref, opt, net, eng = make_pair("lars", channels_last=channels_last, max_grad_norm=thr, accumulation_steps=k)
    assert len(eng.buckets) >= 2 and eng._staged
    for step in range(4):
        if step == 2:
            eng.set_lr(0.2)                                         # mid-run: the device block, no re-capture
            for g in opt.param_groups:
                g["lr"] = 0.2
        x, y = batch(step, BATCH, 200, channels_last)
        want = torch_step(ref, opt, x, y, k, max_norm=thr, lars=LARC)
        eng.train_step(x, y)
        if clipped:
            assert float(eng.last_grad_norm) == pytest.approx(want, rel=1e-5)
        assert float(eng.flat_grad.abs().max()) == 0.0
        close_params(net, ref, 2e-5, step)
        t = eng.last_trust_ratios
        assert t.shape == (len(list(net.parameters())),) and t.dtype == torch.float32
        for ti, p in zip(t.tolist(), net.parameters()):
            assert (ti == 1.0) if p.dim() <= 1 else (0.0 < ti < math.inf and ti != 1.0)
    assert float(eng._hp[0]) == pytest.approx(0.2) and float(eng._hp[4]) == pytest.approx(LARC["trust_coefficient"])


@pytest.mark.parametrize("clipped", [False, True], ids=["unclipped", "clipped"])
@pytest.mark.parametrize("k", [1, 2])
def test_launch_order(cpu_engine, clipped, k):
    eng = make_pair("lars", max_grad_norm=1.0 if clipped else None, accumulation_steps=k)[3]
    nb, comm = len(eng.buckets), eng.comm
    for step in range(2):
        n0, l0 = len(comm.log), comm.launches
        eng.train_step(*batch(step, BATCH, 200))
        kinds = [kind for kind, _ in comm.log[n0:]]
        want = ["norm"] * nb + ["accum"] * nb * (k - 1) + (["coef"] if clipped else [])
        want += ["lars_norm"] * nb + ["lars_trust"] + ["lars_apply"] * nb
        assert kinds == want                                        # (no bare barrier: the trust kernel's stands for it)
        assert comm.launches - l0 == len(want)
        assert [n for kind, n in comm.log[n0:] if kind == "lars_apply"] == [b.numel for b in eng.buckets]


def test_other_optimizers_have_no_trust_ratios(cpu_engine):
    for kw in ({}, {"optimizer": "adamw"}):
        eng = BnetDDP(_model(), bucket_mb=0.002, comm=FakeComm(), **kw)
        assert eng.last_trust_ratios is None


def test_bucket_without_gradient_is_left_alone(cpu_engine):
    ref, opt, net, eng = make_pair("lars", model=Branchy)
    idle = [k for k, b in enumerate(eng.buckets) if len(b.params) == 1 and b.params[0] is net.unused.weight]
    assert len(idle) == 1
    w0 = net.unused.weight.detach().clone()
    eng._lars_slots.fill_(7.0)                                       # stale sums must not reach the ratios
    for step in range(2):
        x, y = batch(step, BATCH, 200)
        ref.unused.weight.grad = None
        torch_step(ref, opt, x, y, lars=LARC)
        eng.train_step(x, y)
        close_params(net, ref, 2e-5, step)
    assert torch.equal(net.unused.weight, w0)
    assert float(eng.last_trust_ratios[0]) == 1.0                    # (`unused` is the first parameter)
    assert [kind for kind, _ in eng.comm.log].count("lars_apply") == 2 * (len(eng.buckets) - 1)


def test_state_dict_round_trip_and_keys(cpu_engine):
    eng = make_pair("lars")[3]
    eng.train_step(*batch(0, BATCH, 200))
    state = eng.optimizer_state_dict()
    assert set(state) == {"optimizer", "lr", "momentum", "weight_decay", "trust_coefficient", "eps", "world", "rank", "buckets"}
    assert state["optimizer"] == "lars" and all(set(b) == {"master", "momentum"} for b in state["buckets"])
    resumed = make_pair("lars")[3]
    resumed.load_optimizer_state_dict(copy.deepcopy(state))
    for b1, b2 in zip(resumed.buckets, eng.buckets):
        assert all(torch.equal(t1, t2) for t1, t2 in zip(b1.state, b2.state))
    assert torch.equal(resumed._hp, eng._hp)
    for other in ({}, {"optimizer": "adamw"}):
        plain = BnetDDP(_model(), bucket_mb=0.002, comm=FakeComm(), **other)
        with pytest.raises(ValueError):
            plain.load_optimizer_state_dict(copy.deepcopy(state))
        with pytest.raises(ValueError):
            resumed.load_optimizer_state_dict(copy.deepcopy(plain.optimizer_state_dict()))


def test_rejects_bad_arguments(cpu_engine):
    for bad in ({"trust_coefficient": 0.0}, {"trust_coefficient": -1e-3}, {"trust_coefficient": float("nan")},
                {"eps": -1e-8}, {"eps": float("nan")}, {"amsgrad": True}, {"maximize": True}):
        with pytest.raises(ValueError):
            BnetDDP(_model(), optimizer="lars", bucket_mb=0.002, comm=FakeComm(), **bad)
    with pytest.raises(ValueError):
        BnetDDP(_model(), optimizer="lamb", bucket_mb=0.002, comm=FakeComm())

"""BnetDDP(ema_decay=...)'s HOST logic on the CPU: the EMA of the master weights against a float64
torch.optim.swa_utils.AveragedModel (SGD, AdamW and LARS, every 1 and 3, k = 1 and 2, clipped and unclipped), a bucket
without gradient, set_ema_decay and reset_ema mid-run, the launch order, ema_parameters(), the state dict and its
cross-loading rules, an engine without EMA, and every rejected argument.  FakeComm does the kernels' work in plain
PyTorch; the kernels are covered on the GPU by tests/test_ema.py."""
import copy

import pytest
import torch
from engine_fakes import FakeComm, cpu_engine  # noqa: F401 - cpu_engine is a fixture
from engine_fakes import HYPER, LARC, Branchy, batch, make_pair, torch_step
from engine_fakes import small_model as _model
from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn

from bagua_net_b200.parallel.ddp import BnetDDP


BATCH = 8
DECAY = 0.6                  # weights 0.4 (the lerp's first branch) and, after set_ema_decay(0.3), 0.7 (its second)


def _flat_ema(eng):
    return torch.cat([b.ema for b in eng.buckets])        # (one rank: the shards are the buckets, in flat order)


def _as_params(eng, net, flat):
    """`flat` (laid out as flat_param) as one tensor per parameter of `net`."""
    base, es = eng.flat_param.data_ptr(), eng.flat_param.element_size()
    return [flat.as_strided(p.shape, p.stride(), (p.data_ptr() - base) // es) for p in net.parameters()]


def _ema_f64(ema, master, decay, n):
    return master.clone() if n == 0 else torch.lerp(ema, master, 1.0 - decay)


@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("every", [1, 3])
@pytest.mark.parametrize("clipped", [False, True], ids=["unclipped", "clipped"])
@pytest.mark.parametrize("optimizer", ["sgd", "adamw", "lars"])
def test_ema_matches_averaged_model(cpu_engine, optimizer, clipped, every, k):
    thr = 0.05 if clipped else None
    ref, opt, net, eng = make_pair(optimizer, ema_decay=DECAY, ema_every=every, max_grad_norm=thr, accumulation_steps=k)
    avg = AveragedModel(ref, multi_avg_fn=get_ema_multi_avg_fn(DECAY), use_buffers=False)
    assert len(eng.buckets) >= 2
    assert torch.equal(_flat_ema(eng), torch.cat([b.master for b in eng.buckets]))   # a copy of the masters at first
    own = _flat_ema(eng).double()                          # float64 EMA of the engine's own masters
    n = 0
    for step in range(1, 8):
        x, y = batch(step, BATCH, 300)
        torch_step(ref, opt, x, y, k, max_norm=thr, lars=LARC if optimizer == "lars" else None)
        eng.train_step(x, y)
        if step % every == 0:
            avg.update_parameters(ref)
            own = _ema_f64(own, torch.cat([b.master for b in eng.buckets]).double(), DECAY, n)
            n += 1
        assert eng._ema.tolist() == [pytest.approx(1 - DECAY), every, step, n]
        got = _flat_ema(eng)
        assert torch.allclose(got.double(), own, rtol=0, atol=4 * 2.0 ** -24 * float(own.abs().max())), step
        for a, b in zip(_as_params(eng, net, got), avg.module.parameters()):
            assert torch.allclose(a.double(), b, rtol=0, atol=2e-5), (step, float((a.double() - b).abs().max()))
    assert int(avg.n_averaged) == n == 7 // every


@pytest.mark.parametrize("optimizer", ["sgd", "lars"])
def test_bucket_without_gradient_updates_its_ema(cpu_engine, optimizer):
    net, eng = make_pair(optimizer, model=Branchy, ema_decay=DECAY)[2:]
    idle = [b for b in eng.buckets if len(b.params) == 1 and b.params[0] is net.unused.weight]
    assert len(idle) == 1
    idle = idle[0]
    eng.train_step(*batch(0, BATCH, 300))                  # the copy step
    assert torch.equal(idle.ema, idle.master)
    idle.ema.zero_()
    eng.train_step(*batch(1, BATCH, 300))                  # lerp(0, master, 0.4): the bucket's EMA moves without a gradient
    assert torch.equal(idle.ema, torch.lerp(torch.zeros_like(idle.master), idle.master, float(eng._ema[0])))
    assert [kind for kind, _ in eng.comm.log].count("ema_update") == 2 * len(eng.buckets)


def test_set_ema_decay_and_reset_ema_mid_run(cpu_engine):
    ref, opt, net, eng = make_pair("sgd", ema_decay=DECAY, ema_every=2)
    avg = AveragedModel(ref, multi_avg_fn=get_ema_multi_avg_fn(DECAY), use_buffers=False)
    for step in range(1, 11):
        if step == 4:                                      # a decay schedule: weight 0.7, the lerp's other branch
            eng.set_ema_decay(0.3)
            avg.multi_avg_fn = get_ema_multi_avg_fn(0.3)
        if step == 7:                                      # torchvision's n_averaged.fill_(0): the next update copies
            eng.reset_ema()
            avg.n_averaged.fill_(0)
        x, y = batch(step, BATCH, 300)
        torch_step(ref, opt, x, y)
        eng.train_step(x, y)
        if step % 2 == 0:
            avg.update_parameters(ref)
        if step == 8:
            assert torch.equal(_flat_ema(eng), torch.cat([b.master for b in eng.buckets]))   # the copy after the reset
        for a, b in zip(_as_params(eng, net, _flat_ema(eng)), avg.module.parameters()):
            assert torch.allclose(a.double(), b, rtol=0, atol=2e-5), step
    assert eng._ema.tolist() == [pytest.approx(0.7), 2, 10, 2] and int(avg.n_averaged) == 2
    assert eng.ema_decay == 0.3


@pytest.mark.parametrize("k", [1, 2])
@pytest.mark.parametrize("kind", ["sgd", "adamw", "lars", "sgd-clipped"])
def test_launch_order(cpu_engine, kind, k):
    optimizer = kind.split("-")[0]
    eng = make_pair(optimizer, ema_decay=DECAY, ema_every=2, accumulation_steps=k,
                    max_grad_norm=1.0 if "clipped" in kind else None)[3]
    nb, comm = len(eng.buckets), eng.comm
    update = "lars_apply" if optimizer == "lars" else "apply" if k > 1 or "clipped" in kind else optimizer
    for step in range(3):
        n0, l0 = len(comm.log), comm.launches
        eng.train_step(*batch(step, BATCH, 300))
        kinds = [kind for kind, _ in comm.log[n0:]]
        last = max(i for i, kd in enumerate(kinds) if kd == update)
        assert kinds.count(update) == nb                     # one optimizer step per train_step ...
        assert kinds[last + 1:] == ["ema_update"] * nb + ["ema_advance"]   # ... then the EMA, on every step
        assert [n for kd, n in comm.log[n0:] if kd == "ema_update"] == [b.master.numel() for b in eng.buckets]
        assert comm.launches - l0 == len([kd for kd in kinds if kd != "barrier"])
    assert eng._ema.tolist()[2:] == [3, 1]


def test_ema_parameters_publishes_and_restores(cpu_engine):
    for dtype in (torch.float32, torch.bfloat16):
        net = _model().to(dtype)
        eng = BnetDDP(net, bucket_mb=0.002, comm=FakeComm(), **HYPER["sgd"], ema_decay=DECAY, accumulation_steps=2)
        if dtype == torch.float32:
            for step in range(3):
                eng.train_step(*batch(step, BATCH, 300))
        torch.manual_seed(9)
        for b in eng.buckets:                              # an EMA away from the masters, below a bf16 ulp too
            b.ema.copy_(b.master + torch.randn_like(b.master) * 1e-3)
        before = eng.flat_param.clone()
        with eng.ema_parameters() as m:
            assert m is net
            assert torch.equal(eng.flat_param, _flat_ema(eng).to(dtype))
            for p, e in zip(net.parameters(), _as_params(eng, net, _flat_ema(eng))):
                assert torch.equal(p.detach(), e.to(dtype))
            with pytest.raises(ValueError):
                eng.train_step(*batch(0, BATCH, 300))
            with pytest.raises(ValueError):
                eng.finish_step()
            with pytest.raises(ValueError):
                with eng.ema_parameters():
                    pass
        assert torch.equal(eng.flat_param.view(torch.uint8), before.view(torch.uint8))
        if dtype == torch.float32:                         # in the middle of an accumulation step
            x, y = batch(5, BATCH, 300)
            torch.nn.functional.cross_entropy(net(x[:4]), y[:4]).backward()
            eng.finish_step()
            assert eng.micro_step == 1
            with pytest.raises(ValueError):
                with eng.ema_parameters():
                    pass
    with pytest.raises(ValueError):
        with make_pair("sgd")[3].ema_parameters():
            pass


SGD_KEYS = {"lr", "momentum", "weight_decay", "world", "rank", "buckets"}
EMA_KEYS = {"ema_decay", "ema_every", "ema_step", "ema_n_averaged"}


@pytest.mark.parametrize("optimizer", ["sgd", "adamw", "lars"])
def test_state_dict_round_trip(cpu_engine, optimizer):
    eng = make_pair(optimizer, ema_decay=DECAY, ema_every=2)[3]
    for step in range(5):
        eng.train_step(*batch(step, BATCH, 300))
    state = eng.optimizer_state_dict()
    plain = set(make_pair(optimizer)[3].optimizer_state_dict())
    assert set(state) == plain | EMA_KEYS
    assert (state["ema_decay"], state["ema_every"], state["ema_step"], state["ema_n_averaged"]) == (DECAY, 2, 5, 2)
    assert all("ema" in b and torch.equal(b["ema"], e.ema) for b, e in zip(state["buckets"], eng.buckets))
    resumed = make_pair(optimizer, ema_decay=0.9, ema_every=5)[3]
    resumed.load_optimizer_state_dict(copy.deepcopy(state))
    assert torch.equal(resumed._ema, eng._ema) and (resumed.ema_decay, resumed.ema_every) == (DECAY, 2)
    for b1, b2 in zip(resumed.buckets, eng.buckets):
        assert torch.equal(b1.ema, b2.ema) and all(torch.equal(t1, t2) for t1, t2 in zip(b1.state, b2.state))


def test_state_dict_cross_loading(cpu_engine):
    with_ema = make_pair("sgd", ema_decay=DECAY)[3]
    without = make_pair("sgd")[3]
    for step in range(2):
        with_ema.train_step(*batch(step, BATCH, 300))
        without.train_step(*batch(step, BATCH, 300))
    # an EMA would be dropped silently: refused, and nothing is loaded
    masters = [b.master.clone() for b in without.buckets]
    with pytest.raises(ValueError):
        without.load_optimizer_state_dict(copy.deepcopy(with_ema.optimizer_state_dict()))
    assert all(torch.equal(m, b.master) for m, b in zip(masters, without.buckets))
    # a plain checkpoint into an engine with an EMA: the EMA restarts from the loaded masters
    target = make_pair("sgd", ema_decay=DECAY)[3]
    target.load_optimizer_state_dict(copy.deepcopy(without.optimizer_state_dict()))
    for b, o in zip(target.buckets, without.buckets):
        assert torch.equal(b.master, o.master) and torch.equal(b.ema, o.master)
    assert target._ema.tolist() == [pytest.approx(1 - DECAY), 1, 0, 0]


def test_engine_without_ema_is_unchanged(cpu_engine):
    eng = make_pair("sgd")[3]
    assert eng.ema_decay is None and eng._ema is None and all(b.ema is None for b in eng.buckets)
    for step in range(2):
        n0, l0 = len(eng.comm.log), eng.comm.launches
        eng.train_step(*batch(step, BATCH, 300))
        assert [kind for kind, _ in eng.comm.log[n0:]] == ["sgd"] * len(eng.buckets)
        assert eng.comm.launches - l0 == len(eng.buckets)
    state = eng.optimizer_state_dict()
    assert set(state) == SGD_KEYS and all(set(b) == {"master", "momentum"} for b in state["buckets"])
    for call in (lambda: eng.set_ema_decay(0.9), eng.reset_ema):
        with pytest.raises(ValueError):
            call()


def test_rejects_bad_arguments(cpu_engine):
    for bad in ({"ema_decay": -0.1}, {"ema_decay": 1.5}, {"ema_decay": float("nan")}, {"ema_decay": float("inf")},
                {"ema_decay": "x"}, {"ema_decay": [0.9]}, {"ema_decay": 0.9, "ema_every": 0},
                {"ema_decay": 0.9, "ema_every": -3}, {"ema_decay": 0.9, "ema_every": 2.0}, {"ema_decay": 0.9, "ema_every": True},
                {"ema_decay": 0.9, "ema_every": "2"}, {"ema_decay": 0.9, "ema_every": (1 << 24) + 1}):
        with pytest.raises(ValueError):
            make_pair("sgd", **bad)
    eng = make_pair("sgd", ema_decay=0.0)[3]               # the ends of [0, 1] are allowed
    make_pair("sgd", ema_decay=1, ema_every=1 << 24)
    for bad in (-1e-9, 1.0000001, float("nan"), None):
        with pytest.raises(ValueError):
            eng.set_ema_decay(bad)
    assert eng.ema_decay == 0.0 and float(eng._ema[0]) == 1.0

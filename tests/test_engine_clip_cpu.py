"""BnetDDP(max_grad_norm=...)'s HOST logic on the CPU: the three stages of the clipped step (per bucket reduce + sum of
squares from the gradient hook, once per step the norm and the coefficient, per bucket the update from the scratch),
set_max_grad_norm, last_grad_norm, the state dict and the arguments it rejects, against torch.nn.utils.clip_grad_norm_
followed by torch.optim.SGD / AdamW.  FakeComm does the three stages in plain PyTorch; the kernels are covered on the
GPU by tests/test_grad_clip.py."""
import copy
import math

import pytest
import torch
from engine_fakes import FakeComm, cpu_engine  # noqa: F401 - cpu_engine is a fixture
from engine_fakes import Branchy, batch, close_params, make_pair, torch_step
from engine_fakes import small_model as _model

from bagua_net_b200.parallel.ddp import BnetDDP


# thresholds per step: far below the gradient norm (clipped), far above it, inf (norm only), and back
THRESHOLDS = [1e-2, 1e-2, 1e3, math.inf, 1e-2, 1e3]


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
@pytest.mark.parametrize("direct_grads", ["1", "0"], ids=["adopted", "accumulated"])
@pytest.mark.parametrize("channels_last", [True, False])
def test_clipped_engine_trains_like_torch(cpu_engine, optimizer, channels_last, direct_grads):
    cpu_engine.setenv("BNET_DIRECT_GRADS", direct_grads)
    ref, opt, net, eng = make_pair(optimizer, channels_last=channels_last, dtype=torch.float32, max_grad_norm=THRESHOLDS[0])
    assert len(eng.buckets) >= 2
    clipped, kept, wants = [], [], []
    for step, thr in enumerate(THRESHOLDS):
        if thr != eng.max_grad_norm:
            eng.set_max_grad_norm(thr)                          # mid-run, through the device block
        x, y = batch(step, 4, 100, channels_last)
        want = torch_step(ref, opt, x, y, max_norm=thr)
        eng.train_step(x, y)
        got = float(eng.last_grad_norm)
        assert got == pytest.approx(want, rel=1e-5), (step, got, want)
        assert eng.last_grad_norm.dim() == 0 and eng.last_grad_norm.dtype == torch.float32
        kept.append(eng.last_grad_norm)                         # read later: each keeps its own step's norm
        wants.append(want)
        clipped.append(float(eng._clip[2]) < 1.0)
        assert float(eng.flat_grad.abs().max()) == 0.0
        close_params(net, ref, 2e-5, step)
    assert clipped == [True, True, False, False, True, False]
    assert [float(t) for t in kept] == pytest.approx(wants, rel=1e-5) and len(set(float(t) for t in kept)) == len(kept)


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_three_stages_launch_in_order(cpu_engine, optimizer):
    eng = make_pair(optimizer, max_grad_norm=1.0)[3]
    comm = eng.comm
    sizes = sorted(b.numel for b in eng.buckets)
    for step in range(2):
        n0, l0 = len(comm.log), comm.launches
        eng.train_step(*batch(step, 4, 100))
        log = comm.log[n0:]
        nb = len(eng.buckets)
        assert [k for k, _ in log] == ["norm"] * nb + ["coef"] + ["apply"] * nb
        assert sorted(n for _, n in log[:nb]) == sizes                  # one stage 1 per bucket, from the hooks
        assert log[nb] == ("coef", nb)
        assert [n for _, n in log[nb + 1:]] == [b.numel for b in eng.buckets]  # stage 3 in bucket order
        assert comm.launches - l0 == 2 * nb + 1 and eng.kernel_launches == comm.launches
        if optimizer == "adamw":
            assert comm.steps_seen[-nb:] == [float(step)] * nb and float(eng._hp[6]) == step + 1


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_without_clipping_only_the_one_kernel_step_runs(cpu_engine, optimizer):
    eng = make_pair(optimizer)[3]
    assert eng.max_grad_norm is None and eng.last_grad_norm is None and eng._clip is None
    eng.train_step(*batch(0, 4, 100))
    assert [k for k, _ in eng.comm.log] == [optimizer] * len(eng.buckets)
    assert all(b.scratch is None and b.partial is None for b in eng.buckets)
    with pytest.raises(ValueError):
        eng.set_max_grad_norm(1.0)


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_state_dict_keys_are_unchanged(cpu_engine, optimizer):
    plain = make_pair(optimizer)[3]
    clip = make_pair(optimizer, max_grad_norm=0.5)[3]
    clip.train_step(*batch(0, 4, 100))
    a, b = plain.optimizer_state_dict(), clip.optimizer_state_dict()
    assert set(a) == set(b) and [set(x) for x in a["buckets"]] == [set(x) for x in b["buckets"]]
    resumed = make_pair(optimizer, max_grad_norm=0.5)[3]
    resumed.load_optimizer_state_dict(copy.deepcopy(b))
    for b1, b2 in zip(resumed.buckets, clip.buckets):
        for t1, t2 in zip(b1.state, b2.state):
            assert torch.equal(t1, t2)


def test_rejects_bad_thresholds(cpu_engine):
    for bad in (0.0, -1.0, float("nan"), -math.inf):
        with pytest.raises(ValueError):
            BnetDDP(_model(), bucket_mb=0.002, comm=FakeComm(), max_grad_norm=bad)
    eng = BnetDDP(_model(), bucket_mb=0.002, comm=FakeComm(), max_grad_norm=math.inf)
    assert float(eng._clip[0]) == math.inf
    for bad in (0.0, -2.0, float("nan")):
        with pytest.raises(ValueError):
            eng.set_max_grad_norm(bad)
    assert eng.max_grad_norm == math.inf and float(eng._clip[0]) == math.inf


def test_bucket_without_gradients_gets_no_update(cpu_engine):
    ref, opt, net, eng = make_pair("sgd", model=Branchy, dtype=torch.float32, max_grad_norm=0.05)
    w0 = net.unused.weight.detach().clone()
    lonely = [b for b in eng.buckets if len(b.params) == 1 and b.params[0] is net.unused.weight]
    assert len(lonely) == 1
    for step in range(3):
        x, y = batch(step, 4, 100)
        want = torch_step(ref, opt, x, y, max_norm=0.05)
        eng.train_step(x, y)
        assert float(eng.last_grad_norm) == pytest.approx(want, rel=1e-5)
    assert torch.equal(net.unused.weight, w0) and torch.equal(ref.unused.weight, w0)
    assert [k for k, _ in eng.comm.log].count("apply") == 3 * (len(eng.buckets) - 1)
    close_params(net, ref, 2e-5)

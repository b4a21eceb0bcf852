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
from engine_fakes import small_model as _model

from bagua_net_b200.parallel.ddp import BnetDDP


def _batch(step, channels_last=True):
    torch.manual_seed(100 + step)
    x, y = torch.randn(4, 3, 8, 8), torch.randint(0, 10, (4,))
    return (x.contiguous(memory_format=torch.channels_last) if channels_last else x), y


SGD = dict(lr=0.05, momentum=0.9, weight_decay=1e-3)
ADAMW = dict(lr=3e-3, betas=(0.85, 0.99), eps=1e-7, weight_decay=0.05)
# thresholds per step: far below the gradient norm (clipped), far above it, inf (norm only), and back
THRESHOLDS = [1e-2, 1e-2, 1e3, math.inf, 1e-2, 1e3]


def _pair(optimizer, channels_last=True, model=None, **kw):
    ref, net = (model or _model)(channels_last), (model or _model)(channels_last)
    if optimizer == "adamw":
        opt = torch.optim.AdamW(ref.parameters(), **ADAMW)
        eng = BnetDDP(net, optimizer="adamw", bucket_mb=0.002, comm=FakeComm(), **ADAMW, **kw)
    else:
        opt = torch.optim.SGD(ref.parameters(), **SGD)
        eng = BnetDDP(net, bucket_mb=0.002, comm=FakeComm(), **SGD, **kw)
    return ref, net, opt, eng


def _torch_step(ref, opt, x, y, max_norm):
    opt.zero_grad()
    torch.nn.functional.cross_entropy(ref(x), y).backward()
    norm = torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
    opt.step()
    return float(norm)


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
@pytest.mark.parametrize("direct_grads", ["1", "0"], ids=["adopted", "accumulated"])
@pytest.mark.parametrize("channels_last", [True, False])
def test_clipped_engine_trains_like_torch(cpu_engine, optimizer, channels_last, direct_grads):
    cpu_engine.setenv("BNET_DIRECT_GRADS", direct_grads)
    ref, net, opt, eng = _pair(optimizer, channels_last, max_grad_norm=THRESHOLDS[0])
    assert len(eng.buckets) >= 2
    clipped, kept, wants = [], [], []
    for step, thr in enumerate(THRESHOLDS):
        if thr != eng.max_grad_norm:
            eng.set_max_grad_norm(thr)                          # mid-run, through the device block
        x, y = _batch(step, channels_last)
        want = _torch_step(ref, opt, x, y, thr)
        eng.train_step(x, y)
        got = float(eng.last_grad_norm)
        assert got == pytest.approx(want, rel=1e-5), (step, got, want)
        assert eng.last_grad_norm.dim() == 0 and eng.last_grad_norm.dtype == torch.float32
        kept.append(eng.last_grad_norm)                         # read later: each keeps its own step's norm
        wants.append(want)
        clipped.append(float(eng._clip[2]) < 1.0)
        assert float(eng.flat_grad.abs().max()) == 0.0
        for a, b in zip(net.parameters(), ref.parameters()):
            assert torch.allclose(a, b, rtol=0, atol=2e-5), (step, (a - b).abs().max())
    assert clipped == [True, True, False, False, True, False]
    assert [float(t) for t in kept] == pytest.approx(wants, rel=1e-5) and len(set(float(t) for t in kept)) == len(kept)


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_three_stages_launch_in_order(cpu_engine, optimizer):
    ref, net, opt, eng = _pair(optimizer, max_grad_norm=1.0)
    comm = eng.comm
    sizes = sorted(b.numel for b in eng.buckets)
    for step in range(2):
        n0, l0 = len(comm.log), comm.launches
        eng.train_step(*_batch(step))
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
    ref, net, opt, eng = _pair(optimizer)
    assert eng.max_grad_norm is None and eng.last_grad_norm is None and eng._clip is None
    eng.train_step(*_batch(0))
    assert [k for k, _ in eng.comm.log] == [optimizer] * len(eng.buckets)
    assert all(b.scratch is None and b.partial is None for b in eng.buckets)
    with pytest.raises(ValueError):
        eng.set_max_grad_norm(1.0)


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_state_dict_keys_are_unchanged(cpu_engine, optimizer):
    plain = _pair(optimizer)[3]
    clip = _pair(optimizer, max_grad_norm=0.5)[3]
    clip.train_step(*_batch(0))
    a, b = plain.optimizer_state_dict(), clip.optimizer_state_dict()
    assert set(a) == set(b) and [set(x) for x in a["buckets"]] == [set(x) for x in b["buckets"]]
    resumed = _pair(optimizer, max_grad_norm=0.5)[3]
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


class _WithUnused(torch.nn.Module):
    """small_model plus a layer that gets no gradient, registered first: its weight fills a bucket of its own."""

    def __init__(self, channels_last=True):
        super().__init__()
        torch.manual_seed(4)
        self.unused = torch.nn.Linear(32, 32, bias=False)
        self.net = _model(channels_last)

    def forward(self, x):
        return self.net(x)


def test_bucket_without_gradients_gets_no_update(cpu_engine):
    ref, net, opt, eng = _pair("sgd", model=_WithUnused, max_grad_norm=0.05)
    w0 = net.unused.weight.detach().clone()
    lonely = [b for b in eng.buckets if len(b.params) == 1 and b.params[0] is net.unused.weight]
    assert len(lonely) == 1
    for step in range(3):
        x, y = _batch(step)
        want = _torch_step(ref, opt, x, y, 0.05)
        eng.train_step(x, y)
        assert float(eng.last_grad_norm) == pytest.approx(want, rel=1e-5)
    assert torch.equal(net.unused.weight, w0) and torch.equal(ref.unused.weight, w0)
    assert [k for k, _ in eng.comm.log].count("apply") == 3 * (len(eng.buckets) - 1)
    for a, b in zip(net.parameters(), ref.parameters()):
        assert torch.allclose(a, b, rtol=0, atol=2e-5)

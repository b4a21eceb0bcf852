"""BnetDDP(accumulation_steps=k)'s HOST logic on the CPU: per micro-batch a stage 1 per bucket (store on the bucket's first
contribution in the step, add after that), once per step the coefficient (clipping) or a barrier, one update per bucket,
1/(world * k) gradient scaling, AdamW's step count, micro_step, the custom backward + finish_step loop, and the arguments
and calls it rejects.  The reference is a float64 copy of the model trained by torch.optim.SGD / AdamW on the FULL batch
(+ clip_grad_norm_).  FakeComm does the stages in plain PyTorch; the kernels are covered on the GPU by
tests/test_grad_accum.py."""
import copy
import math

import pytest
import torch
from engine_fakes import FakeComm, cpu_engine  # noqa: F401 - cpu_engine is a fixture
from engine_fakes import Branchy, batch, close_params, make_pair, torch_step
from engine_fakes import small_model as _model

from bagua_net_b200.parallel.ddp import BnetDDP


BATCH = 12                                      # divisible by every k tested
# clipping thresholds per step: far below the gradient norm, far above it, inf (norm only), below again
THRESHOLDS = [1e-2, 1e3, math.inf, 1e-2]


@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
@pytest.mark.parametrize("clipped", [False, True], ids=["unclipped", "clipped"])
@pytest.mark.parametrize("direct_grads", ["1", "0"], ids=["adopted", "accumulated"])
@pytest.mark.parametrize("channels_last", [True, False])
def test_accumulating_engine_trains_like_torch_on_the_full_batch(cpu_engine, k, optimizer, clipped, direct_grads,
                                                                 channels_last):
    cpu_engine.setenv("BNET_DIRECT_GRADS", direct_grads)
    ref, opt, net, eng = make_pair(optimizer, channels_last=channels_last, max_grad_norm=THRESHOLDS[0] if clipped else None,
                                   accumulation_steps=k)
    assert len(eng.buckets) >= 2 and eng.accumulation_steps == k
    for step, thr in enumerate(THRESHOLDS):
        if clipped and thr != eng.max_grad_norm:
            eng.set_max_grad_norm(thr)                           # mid-run, through the device block
        if optimizer == "sgd" and step == 2:
            lr = 0.02
            eng.set_lr(lr)                                       # scalar launch arguments -> the device block
            for g in opt.param_groups:
                g["lr"] = lr
        x, y = batch(step, BATCH, 100, channels_last)
        want = torch_step(ref, opt, x, y, max_norm=thr if clipped else None)     # on the full batch
        eng.train_step(x, y)
        assert eng.micro_step == 0
        if clipped:
            assert float(eng.last_grad_norm) == pytest.approx(want, rel=1e-5), (step, float(eng.last_grad_norm), want)
        else:
            assert eng.last_grad_norm is None
        assert float(eng.flat_grad.abs().max()) == 0.0
        close_params(net, ref, 2e-5, step)
    scales = eng.comm.apply_scales
    assert scales and all(s == pytest.approx(1.0 / k) for s in scales)
    if clipped:
        assert eng.comm.coef_scales == [1.0 / k] * len(THRESHOLDS)


def test_train_step_loss_is_the_mean_of_the_micro_batch_losses(cpu_engine):
    ref, opt, net, eng = make_pair("sgd", accumulation_steps=3)
    x, y = batch(0, BATCH, 100)
    with torch.no_grad():
        want = sum(float(torch.nn.functional.cross_entropy(net(xs), ys)) for xs, ys in zip(x.split(4), y.split(4))) / 3
    assert float(eng.train_step(x, y)) == pytest.approx(want, rel=1e-6)


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
@pytest.mark.parametrize("clipped", [False, True], ids=["unclipped", "clipped"])
def test_launch_log_per_micro_batch_and_per_step(cpu_engine, optimizer, clipped):
    k = 3
    ref, opt, net, eng = make_pair(optimizer, max_grad_norm=1.0 if clipped else None, accumulation_steps=k)
    comm, nb = eng.comm, len(eng.buckets)
    sizes = sorted(b.numel for b in eng.buckets)
    for step in range(2):
        n0, l0 = len(comm.log), comm.launches
        eng.train_step(*batch(step, BATCH, 100))
        log = comm.log[n0:]
        stage2 = "coef" if clipped else "barrier"
        assert [kind for kind, _ in log] == ["norm"] * nb + ["accum"] * nb * (k - 1) + [stage2] + ["apply"] * nb
        for m in range(k):                                       # every micro-batch: one stage 1 per bucket
            assert sorted(n for _, n in log[m * nb:(m + 1) * nb]) == sizes
        assert [n for _, n in log[k * nb + 1:]] == [b.numel for b in eng.buckets]
        assert comm.launches - l0 == k * nb + nb + (1 if clipped else 0) and eng.kernel_launches == comm.launches
        if optimizer == "adamw":                                 # the step count advances once per optimizer step
            assert comm.steps_seen[-nb:] == [float(step)] * nb and float(eng._hp[6]) == step + 1
            assert len(comm.steps_seen) == (step + 1) * nb


@pytest.mark.parametrize("clipped", [False, True], ids=["unclipped", "clipped"])
@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_one_micro_batch_keeps_the_old_step(cpu_engine, optimizer, clipped):
    """accumulation_steps=1 issues exactly the calls an engine without the argument issues, with the same scales."""
    logs = []
    for kw in ({}, {"accumulation_steps": 1}):
        ref, opt, net, eng = make_pair(optimizer, max_grad_norm=0.5 if clipped else None, **kw)
        for step in range(2):
            eng.train_step(*batch(step, 4, 100))
        logs.append((eng.comm.log, eng.comm.coef_scales, eng.comm.apply_scales, [p.detach().clone() for p in net.parameters()]))
        nb = len(eng.buckets)
        if clipped:
            assert [kind for kind, _ in eng.comm.log] == (["norm"] * nb + ["coef"] + ["apply"] * nb) * 2
        else:
            assert [kind for kind, _ in eng.comm.log] == [optimizer] * nb * 2
            assert all(b.scratch is None for b in eng.buckets)
    assert logs[0][:3] == logs[1][:3]
    assert all(torch.equal(a, b) for a, b in zip(logs[0][3], logs[1][3]))


@pytest.mark.parametrize("clipped", [False, True], ids=["unclipped", "clipped"])
def test_bucket_first_fed_in_the_second_micro_batch_stores_and_an_idle_bucket_is_left_alone(cpu_engine, clipped):
    """A custom backward + finish_step loop; the reference is torch's own accumulation (loss / k per micro-batch) in float64.
    `late` gets its first gradient in micro-batch 2 (stored, not added to a stale scratch), `unused` none in the step
    (no update, nothing in the norm)."""
    k, thr = 3, (0.05 if clipped else None)
    ref, opt, net, eng = make_pair("sgd", model=lambda cl: Branchy(cl, late=True), max_grad_norm=thr, accumulation_steps=k)
    late = [b for b in eng.buckets if len(b.params) == 1 and b.params[0] is net.late.weight]
    idle = [b for b in eng.buckets if len(b.params) == 1 and b.params[0] is net.unused.weight]
    assert len(late) == 1 and len(idle) == 1
    late, idle = late[0], idle[0]
    w0 = net.unused.weight.detach().clone()
    late.scratch.fill_(1e6)                                      # stale: must be overwritten, not added to
    for step in range(3):
        x, y = batch(step, BATCH, 100)
        opt.zero_grad()
        n0 = len(eng.comm.log)
        for m, (xs, ys) in enumerate(zip(x.split(BATCH // k), y.split(BATCH // k))):
            assert eng.micro_step == m
            net.use_late = ref.use_late = (m >= 1)
            torch.nn.functional.cross_entropy(net(xs), ys).backward()
            eng.finish_step()
            (torch.nn.functional.cross_entropy(ref(xs.double()), ys) / k).backward()
        want = float(torch.nn.utils.clip_grad_norm_(ref.parameters(), thr if clipped else math.inf))
        opt.step()
        late_calls = [kind for kind, n in eng.comm.log[n0:] if n == late.numel and kind in ("norm", "accum")]
        assert late_calls == ["norm", "accum"]                   # micro-batch 2 stores, micro-batch 3 adds
        if clipped:
            assert float(eng.last_grad_norm) == pytest.approx(want, rel=1e-5)
        close_params(net, ref, 2e-5, step)
    assert torch.equal(net.unused.weight, w0)
    assert [kind for kind, _ in eng.comm.log].count("apply") == 3 * (len(eng.buckets) - 1)
    assert float(idle.partial.abs().max()) == 0.0


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_custom_loop_matches_train_step(cpu_engine, optimizer):
    k = 4
    a = make_pair(optimizer, max_grad_norm=0.1, accumulation_steps=k)
    b = make_pair(optimizer, max_grad_norm=0.1, accumulation_steps=k)
    for step in range(3):
        x, y = batch(step, BATCH, 100)
        a[3].train_step(x, y)
        for m, (xs, ys) in enumerate(zip(x.split(BATCH // k), y.split(BATCH // k))):
            assert b[3].micro_step == m
            torch.nn.functional.cross_entropy(b[2](xs).float(), ys).backward()
            b[3].finish_step()
        assert b[3].micro_step == 0
        for p, q in zip(a[2].parameters(), b[2].parameters()):
            assert torch.equal(p, q)
        for ba, bb in zip(a[3].buckets, b[3].buckets):
            assert all(torch.equal(s, t) for s, t in zip(ba.state, bb.state))
        assert torch.equal(a[3].last_grad_norm, b[3].last_grad_norm)
    assert a[3].comm.log == b[3].comm.log


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_checkpoint_at_step_boundaries_only(cpu_engine, optimizer):
    ref, opt, net, eng = make_pair(optimizer, accumulation_steps=2)
    plain = make_pair(optimizer)[3]
    eng.train_step(*batch(0, BATCH, 100))
    state = eng.optimizer_state_dict()
    assert set(state) == set(plain.optimizer_state_dict())
    assert [set(s) for s in state["buckets"]] == [set(s) for s in plain.optimizer_state_dict()["buckets"]]
    x, y = batch(1, BATCH, 100)
    torch.nn.functional.cross_entropy(net(x[:6]), y[:6]).backward()
    eng.finish_step()
    assert eng.micro_step == 1
    with pytest.raises(ValueError):
        eng.optimizer_state_dict()
    with pytest.raises(ValueError):
        eng.load_optimizer_state_dict(copy.deepcopy(state))
    with pytest.raises(ValueError):
        eng.train_step(x, y)                                     # in the middle of a step
    torch.nn.functional.cross_entropy(net(x[6:]), y[6:]).backward()
    eng.finish_step()
    assert eng.micro_step == 0
    resumed = make_pair(optimizer, accumulation_steps=2)[3]
    resumed.load_optimizer_state_dict(copy.deepcopy(eng.optimizer_state_dict()))
    for b1, b2 in zip(resumed.buckets, eng.buckets):
        assert all(torch.equal(t1, t2) for t1, t2 in zip(b1.state, b2.state))


def test_rejects_bad_arguments(cpu_engine):
    for bad in (0, -1, 1.5, 2.0, "2", None, True):
        with pytest.raises(ValueError):
            BnetDDP(_model(), bucket_mb=0.002, comm=FakeComm(), accumulation_steps=bad)
    eng = BnetDDP(_model(), bucket_mb=0.002, comm=FakeComm(), accumulation_steps=4)
    for n in (6, 10, 3):
        x, y = batch(0, n, 100)
        with pytest.raises(ValueError):
            eng.train_step(x, y)
    x, y = batch(0, 8, 100)
    with pytest.raises(ValueError):
        eng.train_step(x, y[:4])
    assert eng.micro_step == 0 and eng.comm.log == []
    eng.train_step(x, y)
    assert eng.micro_step == 0


def test_micro_batches_of_a_channels_last_batch_stay_channels_last(cpu_engine):
    seen = []

    class Spy(torch.nn.Module):
        def __init__(self, channels_last=True):
            super().__init__()
            self.net = _model(channels_last)

        def forward(self, x):
            seen.append((x.shape[0], x.is_contiguous(memory_format=torch.channels_last)))
            return self.net(x)

    eng = BnetDDP(Spy(), bucket_mb=0.002, comm=FakeComm(), accumulation_steps=3)
    eng.train_step(*batch(0, BATCH, 100))
    assert seen == [(4, True)] * 3

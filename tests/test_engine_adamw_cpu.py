"""BnetDDP(optimizer="adamw")'s HOST logic on the CPU: the per-bucket launches of the fused all-reduce + AdamW step, the
device-side hyper-parameter block and its step count, set_lr, optimizer state save / load, and the arguments it rejects.
The symmetric heap and the fused kernel are replaced by a fake comm whose `fused_allreduce_adamw` is the same arithmetic
in plain PyTorch (world size 1), and the CUDA stream / event calls by stubs — bagua_net_b200/parallel/ddp.py itself runs
unmodified.  The kernel is covered on the GPU by tests/test_fused_adamw.py."""
import contextlib
import copy
import math

import pytest
import torch

from bagua_net_b200.parallel.ddp import BnetDDP


class FakeStream:
    def wait_event(self, ev):
        pass

    def wait_stream(self, s):
        pass

    def synchronize(self):
        pass


class FakeEvent:
    def record(self, s=None):
        pass


class FakeComm:
    """What BnetDDP needs from SymmComm, for one rank, in host memory."""

    def __init__(self):
        self.world, self.rank, self.launches = 1, 0, 0
        self.steps_seen = []               # the step count every fused launch read

    def alloc(self, numel, dtype):
        return torch.zeros(numel, dtype=dtype)

    def all_reduce(self, t, op="sum", **kw):
        return t

    def fused_allreduce_sgd(self, grad, param, master, mom, lr, momentum, weight_decay, grad_scale=None, zero_grads=True,
                            channel=0, nblocks=0, stream=None, hp=None):
        if hp is not None:
            lr, momentum, weight_decay, scale = (float(v) for v in hp[:4])
        else:
            scale = 1.0 / self.world if grad_scale is None else grad_scale
        mom.mul_(momentum).add_(grad.float() * scale + weight_decay * master)
        master.sub_(lr * mom)
        param.copy_(master.to(param.dtype))
        if zero_grads:
            grad.zero_()
        self.launches += 1

    def fused_allreduce_adamw(self, grad, param, master, exp_avg, exp_avg_sq, hp, zero_grads=True, channel=0, nblocks=0,
                              stream=None):
        assert hp.dtype == torch.float32 and hp.numel() == 8
        lr, b1, b2, eps, wd, scale, step = (float(v) for v in hp[:7])
        t = step + 1
        g = grad.float() * scale
        master.mul_(1 - lr * wd)
        exp_avg.mul_(b1).add_(g, alpha=1 - b1)
        exp_avg_sq.mul_(b2).addcmul_(g, g, value=1 - b2)
        denom = (exp_avg_sq.sqrt() / math.sqrt(1 - b2 ** t)).add_(eps)
        master.addcdiv_(exp_avg, denom, value=-lr / (1 - b1 ** t))
        param.copy_(master.to(param.dtype))
        if zero_grads:
            grad.zero_()
        self.launches += 1
        self.steps_seen.append(step)


@pytest.fixture
def cpu_engine(monkeypatch):
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "Event", lambda *a, **k: FakeEvent())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    return monkeypatch


def _model(channels_last=True):
    torch.manual_seed(3)
    m = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.ReLU(), torch.nn.Conv2d(8, 8, 3, padding=1), torch.nn.ReLU(),
                            torch.nn.AdaptiveAvgPool2d(2), torch.nn.Flatten(), torch.nn.Linear(32, 10))
    return m.to(memory_format=torch.channels_last) if channels_last else m


def _batch(step, channels_last=True):
    torch.manual_seed(100 + step)
    x, y = torch.randn(4, 3, 8, 8), torch.randint(0, 10, (4,))
    return (x.contiguous(memory_format=torch.channels_last) if channels_last else x), y


HYPER = dict(lr=3e-3, betas=(0.85, 0.99), eps=1e-7, weight_decay=0.05)


@pytest.mark.parametrize("direct_grads", ["1", "0"], ids=["adopted", "accumulated"])
@pytest.mark.parametrize("channels_last", [True, False])
def test_engine_trains_like_torch_adamw(cpu_engine, channels_last, direct_grads):
    cpu_engine.setenv("BNET_DIRECT_GRADS", direct_grads)
    ref, net = _model(channels_last), _model(channels_last)
    opt = torch.optim.AdamW(ref.parameters(), **HYPER)
    comm = FakeComm()
    eng = BnetDDP(net, optimizer="adamw", bucket_mb=0.002, comm=comm, **HYPER)   # ~2 KB buckets: several of them
    assert len(eng.buckets) >= 2 and eng._hp is not None
    for step in range(6):
        if step == 3:                                          # a learning-rate schedule step mid-run
            eng.set_lr(1e-3, weight_decay=0.02)
            for g in opt.param_groups:
                g["lr"], g["weight_decay"] = 1e-3, 0.02
        x, y = _batch(step, channels_last)
        opt.zero_grad()
        l_ref = torch.nn.functional.cross_entropy(ref(x), y)
        l_ref.backward()
        l_ref = l_ref.detach()
        opt.step()
        n0 = len(comm.steps_seen)
        l_eng = eng.train_step(x, y)
        # one fused launch per bucket, all reading this step's count; the count advances once per step
        assert comm.steps_seen[n0:] == [float(step)] * len(eng.buckets)
        assert float(eng._hp[6]) == step + 1
        assert abs(float(l_eng) - float(l_ref)) < 1e-5, (step, float(l_eng), float(l_ref))
        assert float(eng.flat_grad.abs().max()) == 0.0
    for a, b in zip(net.parameters(), ref.parameters()):
        assert torch.allclose(a, b, rtol=0, atol=1e-5), (a - b).abs().max()
    for p in ref.parameters():                                 # (the engine's moments are torch's, shard by shard)
        assert opt.state[p]["step"] == 6
    assert eng.kernel_launches == 6 * len(eng.buckets)


def test_optimizer_state_round_trip_continues_bit_identically(cpu_engine):
    comm = FakeComm()
    net = _model()
    eng = BnetDDP(net, optimizer="adamw", bucket_mb=0.002, comm=comm, **HYPER)
    for step in range(3):
        eng.train_step(*_batch(step))
    weights = copy.deepcopy(net.state_dict())
    state = copy.deepcopy(eng.optimizer_state_dict())
    assert state["optimizer"] == "adamw" and state["step"] == 3 and state["betas"] == HYPER["betas"]
    assert state["eps"] == HYPER["eps"] and set(state["buckets"][0]) == {"master", "exp_avg", "exp_avg_sq"}
    for step in range(3, 5):
        eng.train_step(*_batch(step))
    fresh = _model()
    fresh.load_state_dict(weights)
    other = BnetDDP(fresh, optimizer="adamw", lr=0.5, betas=(0.5, 0.5), eps=1.0, bucket_mb=0.002, comm=FakeComm())
    other.load_optimizer_state_dict(state)
    assert float(other._hp[6]) == 3.0 and other.betas == HYPER["betas"] and other.lr == HYPER["lr"]
    for step in range(3, 5):
        other.train_step(*_batch(step))
    assert torch.equal(other.flat_param, eng.flat_param)
    for b1, b2 in zip(other.buckets, eng.buckets):
        for t1, t2 in zip(other._state(b1), eng._state(b2)):
            assert torch.equal(t1, t2)


def test_adamw_rejects_what_it_does_not_offer(cpu_engine):
    with pytest.raises(ValueError):
        BnetDDP(_model(), optimizer="lamb", comm=FakeComm())
    with pytest.raises(ValueError):
        BnetDDP(_model(), optimizer="adamw", amsgrad=True, comm=FakeComm())
    with pytest.raises(ValueError):
        BnetDDP(_model(), optimizer="adamw", maximize=True, comm=FakeComm())
    with pytest.raises(ValueError):
        BnetDDP(_model(), optimizer="adamw", momentum=0.9, comm=FakeComm())
    with pytest.raises(ValueError):
        BnetDDP(_model(), optimizer="adamw", betas=(0.9, 1.0), comm=FakeComm())
    adamw = BnetDDP(_model(), optimizer="adamw", bucket_mb=0.002, comm=FakeComm())
    sgd = BnetDDP(_model(), bucket_mb=0.002, comm=FakeComm())
    with pytest.raises(ValueError):
        adamw.set_lr(0.1, momentum=0.9)
    with pytest.raises(ValueError):
        adamw.load_optimizer_state_dict(copy.deepcopy(sgd.optimizer_state_dict()))
    with pytest.raises(ValueError):
        sgd.load_optimizer_state_dict(copy.deepcopy(adamw.optimizer_state_dict()))


def test_sgd_engine_is_unchanged(cpu_engine):
    comm = FakeComm()
    eng = BnetDDP(_model(), lr=0.1, weight_decay=1e-4, bucket_mb=0.002, comm=comm)
    assert eng.optimizer == "sgd" and eng.momentum == 0.9 and getattr(eng, "_hp", None) is None
    eng.train_step(*_batch(0))
    assert comm.steps_seen == [] and comm.launches == len(eng.buckets)
    state = eng.optimizer_state_dict()
    assert set(state) == {"lr", "momentum", "weight_decay", "world", "rank", "buckets"}
    assert all(set(b) == {"master", "momentum"} for b in state["buckets"])
    eng.set_lr(0.05, momentum=0.8)
    assert eng._hp.tolist() == pytest.approx([0.05, 0.8, 1e-4, 1.0])

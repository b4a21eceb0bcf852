"""What the CPU tests of BnetDDP's host logic put in place of the GPU: a comm whose fused SGD and AdamW steps are the same
arithmetic in plain PyTorch (one rank, host memory), stubs for the CUDA stream / event calls (the `cpu_engine` fixture)
and a small model.  bagua_net_b200/parallel/ddp.py itself runs unmodified."""
import contextlib
import math

import pytest
import torch


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
        self.calls = []                    # the gradient numel of every fused launch
        self.steps_seen = []               # the step count every fused AdamW launch read

    def alloc(self, numel, dtype):
        return torch.zeros(numel, dtype=dtype)

    def all_reduce(self, t, op="sum", **kw):
        return t

    def fused_allreduce_sgd(self, grad, param, master, mom, lr, momentum, weight_decay, grad_scale=None, zero_grads=True, channel=0,
                            nblocks=0, stream=None, hp=None):
        if hp is not None:
            lr, momentum, weight_decay, scale = (float(v) for v in hp[:4])
        else:
            scale = 1.0 / self.world if grad_scale is None else grad_scale
        g = grad.float() * scale + weight_decay * master          # mean gradient + L2 term on the fp32 master weights
        mom.mul_(momentum).add_(g)
        master.sub_(lr * mom)
        param.copy_(master.to(param.dtype))
        if zero_grads:
            grad.zero_()
        self.launches += 1
        self.calls.append(grad.numel())

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
        self.calls.append(grad.numel())
        self.steps_seen.append(step)


@pytest.fixture
def cpu_engine(monkeypatch):
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "Event", lambda *a, **k: FakeEvent())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    return monkeypatch


def small_model(channels_last=True):
    torch.manual_seed(3)
    m = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.ReLU(), torch.nn.Conv2d(8, 8, 3, padding=1), torch.nn.ReLU(),
                            torch.nn.AdaptiveAvgPool2d(2), torch.nn.Flatten(), torch.nn.Linear(32, 10))
    return m.to(memory_format=torch.channels_last) if channels_last else m

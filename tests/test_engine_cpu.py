"""The fused data-parallel engine's HOST logic on the CPU: bucket planning, the flat parameter / gradient views (including
channels_last filters), the hook-driven launches of the per-bucket "collective + optimizer" step, finish_step, learning-rate
changes, optimizer state save / load.  The symmetric heap, the fused kernel and the CUDA stream / event calls are replaced
by the stand-ins of tests/engine_fakes.py.  The device side is covered by the GPU tests (tests/test_gpu.py:
`test_ddp_engine_*`, `test_fused_sgd_*`)."""
import copy

import pytest
import torch
from engine_fakes import FakeComm, cpu_engine  # noqa: F401 - cpu_engine is a fixture
from engine_fakes import close_params, torch_step
from engine_fakes import small_model as _model

from bagua_net_b200.parallel import ddp as ddp_mod
from bagua_net_b200.parallel.ddp import BnetDDP, plan_buckets


def test_plan_buckets_covers_every_parameter_once():
    numels = [1000, 24, 5_000_000, 7, 300_000, 64]
    plan, total = plan_buckets(numels, 2, 8, 1.0)                # 1 MB buckets, 8 ranks
    seen = sorted(pi for _, _, members in plan for pi, _ in members)
    assert seen == list(range(len(numels)))
    end = 0
    for start, numel, members in plan:
        assert start == end and numel % (8 * 8) == 0            # contiguous buckets, each divisible into 16-byte vectors per rank
        offs = sorted(off for _, off in members)
        assert offs[0] >= start and all(o < start + numel for o in offs)
        end = start + numel
    assert end == total >= sum(numels)


@pytest.mark.parametrize("channels_last", [True, False])
def test_engine_trains_like_torch_sgd(cpu_engine, channels_last):
    lr, mom, wd = 0.05, 0.9, 1e-3
    ref = _model(channels_last)
    eng_model = _model(channels_last)
    eng_model.load_state_dict(ref.state_dict())
    opt = torch.optim.SGD(ref.parameters(), lr=lr, momentum=mom, weight_decay=wd)
    comm = FakeComm()
    eng = BnetDDP(eng_model, lr=lr, momentum=mom, weight_decay=wd, bucket_mb=0.002, comm=comm)   # ~2 KB buckets: several of them
    assert len(eng.buckets) >= 2
    # parameters now live in the flat buffer, filters keep their memory format
    for p in eng_model.parameters():
        assert p.data_ptr() >= eng.flat_param.data_ptr() and p.data_ptr() < eng.flat_param.data_ptr() + eng.flat_param.numel() * 4
        if p.dim() == 4 and channels_last:
            assert p.is_contiguous(memory_format=torch.channels_last)
    x = torch.randn(4, 3, 8, 8)
    y = torch.randint(0, 10, (4,))
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    for step in range(4):
        with torch.no_grad():
            l_ref = float(torch.nn.functional.cross_entropy(ref(x), y))
        torch_step(ref, opt, x, y)
        n0 = comm.launches
        l_eng = eng.train_step(x, y)
        assert comm.launches - n0 == len(eng.buckets)           # one fused launch per bucket per step
        assert abs(float(l_eng.detach()) - l_ref) < 1e-5, (step, float(l_eng.detach()), l_ref)
        assert float(eng.flat_grad.abs().max()) == 0.0            # gradients are handed back zeroed
    close_params(eng_model, ref, 1e-5, rtol=1e-5)
    assert eng.kernel_launches == 4 * len(eng.buckets)


class _LinearDirect(torch.autograd.Function):
    """A linear layer whose backward uses ops.tc_linear.weight_grad (its library path: torch.mm with out=): what the wgmma
    classifier does on a GPU, minus the kernel."""

    @staticmethod
    def forward(ctx, x, w, b):
        ctx.save_for_backward(x, w)
        return x @ w.t() + b

    @staticmethod
    def backward(ctx, gy):
        from bagua_net_b200.ops.tc_linear import weight_grad

        x, w = ctx.saved_tensors
        return gy @ w, weight_grad(gy.contiguous(), x, w, tc=False), gy.sum(0)


class _DirectNet(torch.nn.Module):
    def __init__(self, direct):
        super().__init__()
        torch.manual_seed(5)
        self.conv = torch.nn.Conv2d(3, 8, 3, padding=1)
        self.fc1 = torch.nn.Linear(8 * 16, 64)
        self.fc2 = torch.nn.Linear(64, 10)
        self.direct = direct

    def forward(self, x):
        h = torch.relu(self.conv(x))
        h = torch.nn.functional.adaptive_avg_pool2d(h, 4).flatten(1)
        lin = (lambda m, t: _LinearDirect.apply(t, m.weight, m.bias)) if self.direct else (lambda m, t: m(t))
        return lin(self.fc2, torch.relu(lin(self.fc1, h)))


def test_producers_that_write_into_their_gradient_slice_are_adopted_without_a_copy(cpu_engine):
    """The gradient path of the engine: p.grad is None before backward; a producer that looked its slice up and wrote there
    hands back a tensor over that memory and autograd adopts it (no add, no copy); every other gradient is copied into its
    slice by the hook.  Either way the training trajectory is torch.optim.SGD's."""
    lr, mom, wd = 0.05, 0.9, 1e-3
    x, y = torch.randn(6, 3, 8, 8), torch.randint(0, 10, (6,))
    ref = _DirectNet(direct=False)
    opt = torch.optim.SGD(ref.parameters(), lr=lr, momentum=mom, weight_decay=wd)
    copies = {}
    for direct in (False, True):
        net = _DirectNet(direct=direct)
        net.load_state_dict(_DirectNet(direct=False).state_dict())
        eng = BnetDDP(net, lr=lr, momentum=mom, weight_decay=wd, bucket_mb=0.002, comm=FakeComm())
        assert all(p.grad is None for p in net.parameters())
        ref.load_state_dict(_DirectNet(direct=False).state_dict())
        opt = torch.optim.SGD(ref.parameters(), lr=lr, momentum=mom, weight_decay=wd)
        for _ in range(3):
            torch_step(ref, opt, x, y)
            eng.train_step(x, y)
            assert all(p.grad is None for p in net.parameters())          # nothing lingers between steps
        close_params(net, ref, 1e-5, direct, rtol=1e-5)
        copies[direct] = eng.grad_copies
    # a registration dies with its owner (an engine lives as long as the model its hooks sit on; once both are gone the
    # buffers may be unmapped and the addresses reused)
    import gc

    from bagua_net_b200.ops import grad_target

    class Owner:
        pass

    o, wt, slot = Owner(), torch.zeros(4, 4), torch.zeros(4, 4)
    grad_target.register(wt, slot, owner=o)
    assert grad_target.lookup(wt, shape=(2, 8)) is None and grad_target.lookup(torch.zeros(4, 4)) is None
    assert grad_target.lookup(wt) is slot and grad_target.lookup(wt) is None      # handed out once per backward pass ...
    grad_target.release(wt)
    assert grad_target.lookup(wt) is slot                                         # ... until the engine's hook releases it
    grad_target.release(wt)
    del o
    gc.collect()
    assert grad_target.lookup(wt) is None
    assert grad_target.lookup(net.fc1.weight) is not None                # (the last engine is still alive: its model is)
    grad_target.release(net.fc1.weight)
    nparams = len(list(ref.parameters()))
    assert copies[False] == 3 * nparams                                  # plain autograd: every gradient arrives in its own tensor
    assert copies[True] == 3 * (nparams - 2)                             # the two linear weights were written in place


class _SharedNet(torch.nn.Module):
    """One weight used twice in the graph: the first use writes its gradient into the slice, the second arrives in a tensor of
    its own and autograd adds it to the adopted slice."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(9)
        self.fc = torch.nn.Linear(16, 16)
        self.head = torch.nn.Linear(16, 10)

    def forward(self, x, direct=True):
        lin = (lambda m, t: _LinearDirect.apply(t, m.weight, m.bias)) if direct else (lambda m, t: m(t))
        return self.head(lin(self.fc, torch.relu(lin(self.fc, x))))


def test_shared_weights_still_accumulate(cpu_engine):
    x, y = torch.randn(5, 16), torch.randint(0, 10, (5,))
    net, ref = _SharedNet(), _SharedNet()
    opt = torch.optim.SGD(ref.parameters(), lr=0.1, momentum=0.9)
    eng = BnetDDP(net, lr=0.1, momentum=0.9, weight_decay=0.0, bucket_mb=0.002, comm=FakeComm())
    for _ in range(3):
        opt.zero_grad()
        torch.nn.functional.cross_entropy(ref(x, direct=False), y).backward()
        opt.step()
        eng.train_step(x, y)
    close_params(net, ref, 1e-5, rtol=1e-5)


def test_engine_accumulate_mode_switch(cpu_engine):
    """BNET_DIRECT_GRADS=0: p.grad is the slice itself and autograd accumulates into it (the behaviour up to round 2)."""
    cpu_engine.setenv("BNET_DIRECT_GRADS", "0")
    net, ref = _model(), _model()
    opt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.9)
    eng = BnetDDP(net, lr=0.05, momentum=0.9, weight_decay=0.0, bucket_mb=0.002, comm=FakeComm())
    assert all(p.grad is not None and p.grad.data_ptr() == eng._grad_view[id(p)].data_ptr() for p in net.parameters())
    x, y = torch.randn(4, 3, 8, 8).contiguous(memory_format=torch.channels_last), torch.randint(0, 10, (4,))
    for _ in range(3):
        torch_step(ref, opt, x, y)
        eng.train_step(x, y)
    assert eng.grad_copies == 0
    close_params(net, ref, 1e-5, rtol=1e-5)


def test_engine_lr_schedule_and_optimizer_state(cpu_engine):
    m = _model()
    comm = FakeComm()
    eng = BnetDDP(m, lr=0.1, momentum=0.9, weight_decay=0.0, bucket_mb=0.002, comm=comm)
    x, y = torch.randn(4, 3, 8, 8).contiguous(memory_format=torch.channels_last), torch.randint(0, 10, (4,))
    eng.train_step(x, y)
    state = copy.deepcopy(eng.optimizer_state_dict())          # (on a GPU `.cpu()` copies; in host memory it aliases the live shards)
    assert state["world"] == 1 and len(state["buckets"]) == len(eng.buckets)
    before = eng.flat_param.clone()
    eng.set_lr(0.0)                                             # hyper-parameters move to a device tensor the kernel reads
    eng.train_step(x, y)
    assert torch.equal(eng.flat_param, before)                  # lr = 0: nothing moves (momentum still accumulates)
    eng.set_lr(0.1)
    eng.train_step(x, y)
    assert not torch.equal(eng.flat_param, before)
    # restoring the saved optimizer state and parameters reproduces the same next step
    snap_params = before.clone()
    eng.flat_param.copy_(snap_params)
    eng.load_optimizer_state_dict(state)
    eng.sync_master_from_params()
    eng.load_optimizer_state_dict(state)                        # (sync rebuilt the master from the parameters; momentum from the state)
    eng.train_step(x, y)
    after_a = eng.flat_param.clone()
    eng.flat_param.copy_(snap_params)
    eng.load_optimizer_state_dict(state)
    eng.train_step(x, y)
    assert torch.allclose(eng.flat_param, after_a, atol=1e-6)
    with pytest.raises(ValueError):
        bad = dict(state, world=2)
        eng.load_optimizer_state_dict(bad)


def test_engine_rejects_mixed_dtypes_and_empty_models(cpu_engine):
    with pytest.raises(ValueError):
        BnetDDP(torch.nn.ReLU(), comm=FakeComm())
    m = torch.nn.Sequential(torch.nn.Linear(4, 4), torch.nn.Linear(4, 4).to(torch.bfloat16))
    with pytest.raises(ValueError):
        BnetDDP(m, comm=FakeComm())
    assert ddp_mod.BnetDDP is BnetDDP


def test_direct_grads_self_check_accepts_the_working_path_and_rejects_a_broken_one(cpu_engine):
    """bench.py asks `direct_grads_self_check` before it trusts adopted gradients with the benchmark: the same model trained
    with accumulated and with adopted gradients must receive the same fp32 updates.  Here on the CPU test bed: the real engine
    passes; an engine whose hook loses the gradients that arrive in tensors of their own fails; so does one that raises."""
    from bagua_net_b200.parallel.ddp import direct_grads_self_check

    def batch():
        torch.manual_seed(11)
        return torch.randn(4, 3, 8, 8).contiguous(memory_format=torch.channels_last), torch.randint(0, 10, (4,))

    kw = dict(make_model=_model, make_comm=FakeComm, make_batch=batch, use_graph=False)
    ok, detail = direct_grads_self_check(**kw)
    assert ok and detail["rel_l2_error_of_updates"] < 1e-6 and detail["grad_copies_accumulate"] == 0 and detail["grad_copies_adopt"] > 0
    import os

    assert "BNET_DIRECT_GRADS" not in os.environ

    real = BnetDDP._on_grad

    def lossy(self, p):
        if self._direct_grads and p.dim() == 4:
            p.grad = None                                  # the filter gradients never reach the flat buffer
        return real(self, p)

    cpu_engine.setattr(BnetDDP, "_on_grad", lossy)
    ok, detail = direct_grads_self_check(**kw)
    assert not ok and detail["rel_l2_error_of_updates"] > 0.05

    def broken(self, p):
        if self._direct_grads:
            raise RuntimeError("hook failed")
        return real(self, p)

    cpu_engine.setattr(BnetDDP, "_on_grad", broken)
    ok, detail = direct_grads_self_check(**kw)
    assert not ok and "hook failed" in detail["error"]


def test_fake_comm_takes_the_parameters_of_symm_comm():
    """The CPU stand-in is called as the engine calls SymmComm: every SymmComm method that ddp.py calls on its comm, with
    the same parameter names, order and defaults."""
    import inspect
    import re

    from bagua_net_b200.parallel.comm import SymmComm

    called = {n for n in re.findall(r"\bcomm\.(\w+)", inspect.getsource(ddp_mod)) if callable(getattr(SymmComm, n, None))}
    world_above_one = {"peer_tensor", "broadcast_tensor"}      # only reached at world > 1; FakeComm is one rank
    assert world_above_one < called
    for name in sorted(called - world_above_one):
        want, got = (list(inspect.signature(getattr(c, name)).parameters.values()) for c in (SymmComm, FakeComm))
        assert [(p.name, p.default) for p in got] == [(p.name, p.default) for p in want], name

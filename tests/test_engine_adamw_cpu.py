"""BnetDDP(optimizer="adamw")'s HOST logic on the CPU: the per-bucket launches of the fused all-reduce + AdamW step, the
device-side hyper-parameter block and its step count, set_lr, optimizer state save / load, and the arguments it rejects.
The symmetric heap, the fused kernel and the CUDA stream / event calls are replaced by the stand-ins of
tests/engine_fakes.py.  The kernel is covered on the GPU by tests/test_fused_adamw.py."""
import copy

import pytest
import torch
from engine_fakes import FakeComm, cpu_engine  # noqa: F401 - cpu_engine is a fixture
from engine_fakes import HYPER, batch, close_params, make_pair, torch_step
from engine_fakes import small_model as _model

from bagua_net_b200.parallel.ddp import BnetDDP


@pytest.mark.parametrize("direct_grads", ["1", "0"], ids=["adopted", "accumulated"])
@pytest.mark.parametrize("channels_last", [True, False])
def test_engine_trains_like_torch_adamw(cpu_engine, channels_last, direct_grads):
    cpu_engine.setenv("BNET_DIRECT_GRADS", direct_grads)
    ref, opt, net, eng = make_pair("adamw", channels_last=channels_last, dtype=torch.float32)
    comm = eng.comm
    assert len(eng.buckets) >= 2 and eng._hp is not None
    for step in range(6):
        if step == 3:                                          # a learning-rate schedule step mid-run
            eng.set_lr(1e-3, weight_decay=0.02)
            for g in opt.param_groups:
                g["lr"], g["weight_decay"] = 1e-3, 0.02
        x, y = batch(step, 4, 100, channels_last)
        with torch.no_grad():
            l_ref = torch.nn.functional.cross_entropy(ref(x), y)
        torch_step(ref, opt, x, y)
        n0 = len(comm.steps_seen)
        l_eng = eng.train_step(x, y)
        # one fused launch per bucket, all reading this step's count; the count advances once per step
        assert comm.steps_seen[n0:] == [float(step)] * len(eng.buckets)
        assert float(eng._hp[6]) == step + 1
        assert abs(float(l_eng) - float(l_ref)) < 1e-5, (step, float(l_eng), float(l_ref))
        assert float(eng.flat_grad.abs().max()) == 0.0
    close_params(net, ref, 1e-5)
    for p in ref.parameters():                                 # (the engine's moments are torch's, shard by shard)
        assert opt.state[p]["step"] == 6
    assert eng.kernel_launches == 6 * len(eng.buckets)


def test_optimizer_state_round_trip_continues_bit_identically(cpu_engine):
    comm = FakeComm()
    net = _model()
    eng = BnetDDP(net, optimizer="adamw", bucket_mb=0.002, comm=comm, **HYPER["adamw"])
    for step in range(3):
        eng.train_step(*batch(step, 4, 100))
    weights = copy.deepcopy(net.state_dict())
    state = copy.deepcopy(eng.optimizer_state_dict())
    assert state["optimizer"] == "adamw" and state["step"] == 3 and state["betas"] == HYPER["adamw"]["betas"]
    assert state["eps"] == HYPER["adamw"]["eps"] and set(state["buckets"][0]) == {"master", "exp_avg", "exp_avg_sq"}
    for step in range(3, 5):
        eng.train_step(*batch(step, 4, 100))
    fresh = _model()
    fresh.load_state_dict(weights)
    other = BnetDDP(fresh, optimizer="adamw", lr=0.5, betas=(0.5, 0.5), eps=1.0, bucket_mb=0.002, comm=FakeComm())
    other.load_optimizer_state_dict(state)
    assert float(other._hp[6]) == 3.0 and other.betas == HYPER["adamw"]["betas"] and other.lr == HYPER["adamw"]["lr"]
    for step in range(3, 5):
        other.train_step(*batch(step, 4, 100))
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
    eng.train_step(*batch(0, 4, 100))
    assert comm.steps_seen == [] and comm.launches == len(eng.buckets)
    state = eng.optimizer_state_dict()
    assert set(state) == {"lr", "momentum", "weight_decay", "world", "rank", "buckets"}
    assert all(set(b) == {"master", "momentum"} for b in state["buckets"])
    eng.set_lr(0.05, momentum=0.8)
    assert eng._hp.tolist() == pytest.approx([0.05, 0.8, 1e-4, 1.0])

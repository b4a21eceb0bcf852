"""BnetDDP(param_groups=...)'s HOST logic on the CPU: every rejected argument, the group segment tables at world sizes 1-8
on VGG16's and ResNet-50's real shapes, the device group table after set_lr / set_param_group / a state load, the
state dict, and the engine against torch.optim.SGD / AdamW given the same groups (alone and with clipping, accumulation
and the EMA).  FakeComm does the grouped entry points as plain torch arithmetic per segment; the kernels are covered
on the GPU by tests/test_param_groups.py."""
import copy
import math

import pytest
import torch
from engine_fakes import FakeComm, cpu_engine  # noqa: F401 - cpu_engine is a fixture
from engine_fakes import batch, close_params, torch_step

from bagua_net_b200.parallel.comm import GROUPS_MAX, check_group_segments
from bagua_net_b200.parallel.ddp import BnetDDP, group_segments, no_weight_decay_groups, plan_buckets


def _net():
    torch.manual_seed(3)
    return torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.BatchNorm2d(8), torch.nn.ReLU(),
                               torch.nn.Conv2d(8, 8, 3, padding=1), torch.nn.ReLU(), torch.nn.AdaptiveAvgPool2d(2),
                               torch.nn.Flatten(), torch.nn.Linear(32, 16), torch.nn.ReLU(), torch.nn.Linear(16, 10))


def _groups(net):
    head = list(net[-1].parameters())
    nwd = [p for p in no_weight_decay_groups(net)[0]["params"] if all(p is not q for q in head)]
    return [{"params": nwd, "weight_decay": 0.0}, {"params": head, "lr_scale": 10.0}]


# ------------------------------------------------------------------ rejected arguments
def test_rejected_groups(cpu_engine):
    net = _net()
    ps = list(net.parameters())
    other = torch.nn.Parameter(torch.zeros(3))
    frozen = _net()
    frozen[0].weight.requires_grad_(False)
    cases = [
        ({"params": ps[:1]}, "list of dicts"),
        ([{"params": ps[:1], "lr": 0.1}], "lr_scale"),
        ([{"params": ps[:1], "momentum": 0.5}], "unknown keys"),
        ([{"params": ps[:1], "betas": (0.9, 0.9)}], "unknown keys"),
        ([{"params": ps[:1], "eps": 1e-6}], "unknown keys"),
        ([{"params": ps[:2]}, {"params": ps[1:3]}], "param groups 0 and 1"),
        ([{"params": ps[:1] + ps[:1]}], "param groups 0 and 0"),
        ([{"params": [other]}], "not a trainable parameter"),
        ([{"params": [torch.zeros(3)]}], "not a trainable parameter"),
        ([{"params": []}], "no parameters"),
        ([{"weight_decay": 0.0}], "no 'params'"),
        ([{"params": ps[:1], "weight_decay": -1e-4}], ">= 0"),
        ([{"params": ps[:1], "lr_scale": float("nan")}], ">= 0"),
        ([{"params": ps[:1], "lr_scale": -1.0}], ">= 0"),
        ([{"params": ps[:1], "weight_decay": float("nan")}], ">= 0"),
        ([{"params": ps[:1], "lr_scale": "x"}], "a number"),
    ]
    for groups, msg in cases:
        with pytest.raises(ValueError, match=msg):
            BnetDDP(_net() if groups is None else net, comm=FakeComm(), param_groups=groups)
    with pytest.raises(ValueError, match="not a trainable parameter"):
        BnetDDP(frozen, comm=FakeComm(), param_groups=[{"params": [frozen[0].weight]}])
    with pytest.raises(ValueError, match="'sgd' and 'adamw'"):
        BnetDDP(net, comm=FakeComm(), optimizer="lars", param_groups=[{"params": ps[:1]}])
    many = torch.nn.Sequential(*[torch.nn.Linear(2, 2, bias=False) for _ in range(GROUPS_MAX + 1)])
    mp = list(many.parameters())
    with pytest.raises(ValueError, match="at most 64"):      # 64 listed + the default group
        BnetDDP(many, comm=FakeComm(), param_groups=[{"params": [p]} for p in mp[:GROUPS_MAX]])
    eng = BnetDDP(many, comm=FakeComm(), param_groups=[{"params": [p]} for p in mp[:GROUPS_MAX - 1]])
    assert len(eng.param_groups) == GROUPS_MAX
    with pytest.raises(ValueError, match="not parameters of the module"):
        no_weight_decay_groups(net, names=["nope"])


def test_set_param_group_rejects(cpu_engine):
    net = _net()
    eng = BnetDDP(net, comm=FakeComm(), param_groups=_groups(net))
    for kw in ({"lr_scale": -1.0}, {"weight_decay": float("nan")}):
        with pytest.raises(ValueError):
            eng.set_param_group(0, **kw)
    for i in (3, -1, True):
        with pytest.raises(ValueError, match="does not exist"):
            eng.set_param_group(i, lr_scale=1.0)
    with pytest.raises(ValueError, match="no param groups"):
        BnetDDP(_net(), comm=FakeComm()).set_param_group(0, lr_scale=1.0)
    assert BnetDDP(_net(), comm=FakeComm()).param_groups is None


# ------------------------------------------------------------------ the segment tables on real shapes
def _shapes(name):
    from bagua_net_b200.models import build_model

    with torch.device("meta"):
        m = build_model(name)
    named = [(n, p) for n, p in m.named_parameters() if p.requires_grad]
    return [p.numel() for _, p in named], [p.dim() for _, p in named]


@pytest.mark.parametrize("model", ["vgg16", "resnet50"])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 6, 7, 8])
def test_group_tables_on_real_shapes(model, world):
    numels, dims = _shapes(model)
    # two groups (decay / no decay) and ~10 lr-scale groups x decay / no decay, by position in the model
    variants = [[int(d <= 1) for d in dims], [2 * (i * 10 // len(dims)) + int(d <= 1) for i, d in enumerate(dims)]]
    es, per_vec = 2, 8
    plan, _ = plan_buckets(numels, es, world, 64.0)
    for group_of in variants:
        ngroups = max(group_of) + 1
        for start, numel, members in plan:
            shard = numel // world // per_vec
            owner = {}
            for pi, off in members:
                for v in range((off - start) // per_vec, (off - start + numels[pi] + per_vec - 1) // per_vec):
                    owner[v] = group_of[pi]                      # brute force: the group of every vector of a tensor
            for r in range(world):
                t = group_segments(members, numels, group_of, start, numel, es, world, r)
                check_group_segments(t, shard, ngroups)          # covers the shard exactly once
                assert all(a[2] != b[2] for a, b in zip(t, t[1:])), "adjacent rows of one group"
                for vec0, nvec, g, _ in t:
                    for v in range(vec0, vec0 + nvec):
                        want = owner.get(r * shard + v)
                        assert want is None or want == g, (model, world, r, v)   # (None: padding, either neighbour)


def test_rejected_group_tables():
    good = [[0, 3, 0, 0], [3, 5, 1, 0]]
    check_group_segments(good, 8, 2)
    for bad, ng in (([], 2), ([[0, 3, 0, 0]], 2), ([[1, 7, 0, 0]], 2), ([[0, 3, 0, 0], [2, 6, 1, 0]], 2),
                    ([[0, 3, 0, 0], [4, 4, 1, 0]], 2), ([[0, 3, 0, 0], [3, 0, 1, 0], [3, 5, 1, 0]], 2),
                    ([[0, 3, 0, 0], [3, 5, 2, 0]], 2), ([[0, 3, -1, 0], [3, 5, 1, 0]], 2), ([[0, 9, 0, 0]], 2),
                    (good, 0), (good, GROUPS_MAX + 1)):
        with pytest.raises(ValueError):
            check_group_segments(bad, 8, ng)


# ------------------------------------------------------------------ the device table and the state dict
def _rows(eng):
    return [[float(torch.tensor(eng.lr * g["lr_scale"], dtype=torch.float32)), float(torch.tensor(g["weight_decay"], dtype=torch.float32))]
            for g in eng.param_groups]


def test_device_table_follows_set_lr_set_param_group_and_load(cpu_engine):
    for optimizer in ("sgd", "adamw"):
        net = _net()
        eng = BnetDDP(net, lr=0.1, weight_decay=1e-3, comm=FakeComm(), optimizer=optimizer, param_groups=_groups(net))
        assert [g["lr_scale"] for g in eng.param_groups] == [1.0, 10.0, 1.0]
        assert [g["weight_decay"] for g in eng.param_groups] == [0.0, 1e-3, 1e-3]
        assert sum(len(g["params"]) for g in eng.param_groups) == len(list(net.parameters()))
        assert eng._groups[:, :2].tolist() == _rows(eng) and eng._groups[:, 2:].abs().sum() == 0
        eng.set_lr(0.03, weight_decay=5e-4)
        assert eng._groups[:, :2].tolist() == _rows(eng)
        assert eng._groups[1, 0].item() == float(torch.tensor(0.03 * 10.0, dtype=torch.float32))
        assert eng._groups[1, 1].item() == float(torch.tensor(5e-4, dtype=torch.float32))   # follows the engine
        eng.set_param_group(1, lr_scale=0.5)
        eng.set_param_group(2, weight_decay=0.0)
        assert eng._groups[:, :2].tolist() == _rows(eng) and eng._groups[2, 1].item() == 0.0
        if optimizer == "sgd":
            assert eng._hp.tolist()[1] == pytest.approx(0.9) and eng._hp[3].item() == 1.0
        sd = eng.optimizer_state_dict()
        assert sd["param_groups"][1] == {"params": sd["param_groups"][1]["params"], "lr_scale": 0.5, "weight_decay": None}
        assert sd["param_groups"][2]["weight_decay"] == 0.0
        net2 = _net()
        eng2 = BnetDDP(net2, lr=1.0, comm=FakeComm(), optimizer=optimizer, param_groups=_groups(net2))
        eng2.load_optimizer_state_dict(copy.deepcopy(sd))
        assert eng2.lr == 0.03 and eng2._groups.tolist() == eng._groups.tolist()
        assert eng2.optimizer_state_dict()["param_groups"] == sd["param_groups"]
        # membership differs; groups on one side only
        net3 = _net()
        eng3 = BnetDDP(net3, comm=FakeComm(), optimizer=optimizer, param_groups=no_weight_decay_groups(net3))
        with pytest.raises(ValueError, match="other parameters"):
            eng3.load_optimizer_state_dict(copy.deepcopy(sd))
        plain = BnetDDP(_net(), comm=FakeComm(), optimizer=optimizer)
        with pytest.raises(ValueError, match="disagree on param groups"):
            plain.load_optimizer_state_dict(copy.deepcopy(sd))
        with pytest.raises(ValueError, match="disagree on param groups"):
            eng2.load_optimizer_state_dict(plain.optimizer_state_dict())
        assert "param_groups" not in plain.optimizer_state_dict()


def test_ungrouped_engine_is_unchanged(cpu_engine):
    comm = FakeComm()
    eng = BnetDDP(_net(), comm=comm)
    assert eng._hp is None and eng._groups is None and all(b.gsegs is None for b in eng.buckets)
    x, y = torch.randn(4, 3, 8, 8), torch.randint(0, 10, (4,))
    eng.train_step(x, y)
    assert {k for k, _ in comm.log} == {"sgd"}


# ------------------------------------------------------------------ the engine against torch.optim with the same groups
def _torch_groups(ref, lr, wd):
    """The torch.optim groups equivalent to _groups(): lr = lr * lr_scale, weight_decay fixed or the engine's."""
    g = _groups(ref)
    g[0].update(lr=lr)
    g[1].update(lr=lr * 10.0, weight_decay=wd)
    rest = [p for p in ref.parameters() if all(p is not q for gg in g for q in gg["params"])]
    return g + [{"params": rest, "lr": lr, "weight_decay": wd}]


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
@pytest.mark.parametrize("extra", [{}, {"max_grad_norm": 0.5}, {"accumulation_steps": 2}, {"ema_decay": 0.5},
                                   {"max_grad_norm": 0.5, "accumulation_steps": 2, "ema_decay": 0.5}],
                         ids=["plain", "clip", "accum", "ema", "all"])
def test_engine_matches_torch_optim_with_groups(cpu_engine, optimizer, extra):
    hyper = dict(lr=0.05, momentum=0.9, weight_decay=1e-2) if optimizer == "sgd" else dict(lr=2e-3, betas=(0.9, 0.99), eps=1e-8,
                                                                                            weight_decay=0.05)
    net, ref = _net().eval(), _net().double().eval()          # (eval: BatchNorm statistics need no accumulation rule)
    comm = FakeComm()
    eng = BnetDDP(net, comm=comm, optimizer=optimizer, bucket_mb=0.002, param_groups=_groups(net), **hyper, **extra)
    assert len(eng.buckets) > 1
    k = extra.get("accumulation_steps", 1)
    lr, wd = hyper["lr"], hyper["weight_decay"]
    cls = torch.optim.SGD if optimizer == "sgd" else torch.optim.AdamW
    kw = {"momentum": 0.9} if optimizer == "sgd" else {"betas": (0.9, 0.99), "eps": 1e-8}
    opt = cls(_torch_groups(ref, lr, wd), **kw)
    ema = [p.detach().clone() for p in ref.parameters()]
    for step in range(4):
        if step == 2:                                          # a schedule change and a group change between steps
            lr, wd = 0.5 * lr, 2 * wd
            eng.set_lr(lr, weight_decay=wd)
            eng.set_param_group(1, lr_scale=3.0)
            for g, (glr, gwd) in zip(opt.param_groups, [(lr, 0.0), (lr * 3.0, wd), (lr, wd)]):
                g["lr"], g["weight_decay"] = glr, gwd
        x, y = batch(step, 8, 100, channels_last=False)
        eng.train_step(x, y)
        torch_step(ref, opt, x, y, k, max_norm=extra.get("max_grad_norm"))
        if "ema_decay" in extra:
            with torch.no_grad():
                for e, p in zip(ema, ref.parameters()):
                    e.copy_(p if step == 0 else torch.lerp(e, p, 0.5))
    kinds = {kind for kind, _ in comm.log}
    assert ("apply_groups" if eng._staged else f"{optimizer}_groups") in kinds and not kinds & {"sgd", "adamw", "apply"}
    close_params(net, ref, 1e-5, (optimizer, extra), rtol=1e-4)
    if "ema_decay" in extra:
        with eng.ema_parameters():
            for p, e in zip(net.parameters(), ema):
                assert torch.allclose(p.double(), e, rtol=1e-4, atol=1e-5)


def test_groups_do_not_change_buckets_or_state_layout(cpu_engine):
    net_a, net_b = _net(), _net()
    a = BnetDDP(net_a, comm=FakeComm(), bucket_mb=0.002)
    b = BnetDDP(net_b, comm=FakeComm(), bucket_mb=0.002, param_groups=_groups(net_b))
    assert [(x.start, x.numel, len(x.params)) for x in a.buckets] == [(x.start, x.numel, len(x.params)) for x in b.buckets]
    assert [t.shape for x in a.buckets for t in x.state] == [t.shape for x in b.buckets for t in x.state]
    assert math.isclose(b.param_groups[1]["lr"], 0.1)

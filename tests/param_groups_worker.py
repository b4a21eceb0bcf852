"""Per-rank bodies of the parameter-group GPU tests (launched by tests/test_param_groups.py, one process per GPU)."""
from __future__ import annotations

import math
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from adamw_worker import RANK, WORLD, same_on_every_rank, setup, teardown  # noqa: E402
from grad_accum_worker import PER_RANK, TOL, global_batch, micro_grads, rel_updates, small_net  # noqa: E402

from bagua_net_b200.parallel.ddp import group_segments, plan_buckets  # noqa: E402

NAN = float("nan")
SENTINEL = 1024.0                  # guard value of the buffers the kernels write (exact in bf16)
# odd tensors (one element, less than a vector, one vector, ...), then layouts around the loop tails of 7 and 132 CTAs
NUMELS = [1, 7, 8, 9, 1728, 5, 1000, 65539, 17, 4096, 3, 64]
NBS = (1, 7, 132, 264)
SGD_HP = [0.1, 0.9, 0.0, 1.0 / WORLD]                                       # {lr, momentum, wd, grad_scale}; lr, wd unused
ADAMW_HP = [0.0, 0.9, 0.99, 1e-8, 0.0, 1.0 / WORLD, 3.0, 0.0]               # step 3: bias corrections below 1
GROUPS = [[0.1, 1e-2], [0.3, 0.0], [0.05, 5e-4]]                            # {lr, wd}: decay, no decay, another lr


def bits(t):
    return t.contiguous().view(torch.uint8)


def layouts(per_vec):
    return (NUMELS, [per_vec * (2 * 512 * 132 * WORLD) - 8 * per_vec, 8, 1], [per_vec * (2 * 512 * 7 * WORLD + 1), 3, 24])


def sync():
    torch.cuda.synchronize()
    if WORLD > 1:
        dist.barrier()


class Bucket:
    """One bucket's heap parameters and gradients and this rank's fp32 state (and scratch), each inside guards of PAD
    elements: the written buffers hold SENTINEL there, the read ones NaN.  `run` restores the inputs, launches, checks
    the guards and returns the state shards and this rank's parameter shard."""

    def __init__(self, comm, numel, dtype, nstate):
        self.pad = 16 * WORLD * 8
        p = self.pad
        self.numel, self.shard = numel, numel // WORLD
        self.pbuf, self.gbuf = comm.alloc(numel + 2 * p, dtype), comm.alloc(numel + 2 * p, dtype)
        self.sbufs = [torch.empty(self.shard + 2 * p, device="cuda") for _ in range(nstate + 1)]   # state..., scratch
        self.param, self.grad = self.pbuf[p:p + numel], self.gbuf[p:p + numel]
        self.state = [b[p:p + self.shard] for b in self.sbufs[:-1]]
        self.scratch = self.sbufs[-1][p:p + self.shard]
        g = torch.Generator(device="cuda").manual_seed(7 + RANK + numel)
        self.g0 = (torch.randn(numel, device="cuda", generator=g) * 1e-2).to(dtype)
        self.s0 = [torch.randn(self.shard, device="cuda", generator=g)] + [
            torch.rand(self.shard, device="cuda", generator=g) * 1e-4 for _ in range(nstate - 1)]
        self.c0 = torch.randn(self.shard, device="cuda", generator=g) * 1e-2
        self.p0 = torch.randn(numel, device="cuda", generator=g).to(dtype)

    def run(self, launch):
        p = self.pad
        for b, v in ((self.pbuf, SENTINEL), (self.gbuf, NAN)):
            b.fill_(v)
        for b in self.sbufs[:-1]:
            b.fill_(SENTINEL)
        self.sbufs[-1].fill_(NAN)
        self.param.copy_(self.p0)
        self.grad.copy_(self.g0)
        for t, s in zip(self.state, self.s0):
            t.copy_(s)
        self.scratch.copy_(self.c0)
        sync()
        launch()
        sync()
        for b in [self.pbuf] + self.sbufs[:-1]:
            assert bool((b[:p] == SENTINEL).all() and (b[-p:] == SENTINEL).all()), "guard region overwritten"
        assert bool(self.gbuf[:p].isnan().all() and self.gbuf[-p:].isnan().all() and self.sbufs[-1][:p].isnan().all()
                    and self.sbufs[-1][-p:].isnan().all()), "input guard overwritten"
        assert same_on_every_rank(self.param), "ranks hold different parameters"
        return [t.clone() for t in self.state] + [self.param[RANK * self.shard:(RANK + 1) * self.shard].clone()]


def _oracle(apply_stage):
    """Per group g: the grouped kernel's results on g's elements equal bitwise those of the ungrouped kernel run with g's lr
    and weight decay; with a single group holding everything, equal everywhere."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(512 << 20)
    cases = 0
    coefs = (0.3, 1e-3, 1.0, 0.0, NAN) if apply_stage else (None,)
    for optimizer in ("sgd", "adamw"):
        nstate = 2 if optimizer == "sgd" else 3
        base = SGD_HP if optimizer == "sgd" else ADAMW_HP
        lr_i, wd_i = (0, 2) if optimizer == "sgd" else (0, 4)
        hp = torch.tensor(base, device="cuda")
        for dtype in (torch.float32, torch.bfloat16):
            es = torch.empty((), dtype=dtype).element_size()
            per_vec = 16 // es
            for numels in layouts(per_vec):
                plan, _ = plan_buckets(numels, es, WORLD, 1e9)
                start, numel, members = plan[0]
                bk = Bucket(comm, numel, dtype, nstate)
                clip = torch.tensor([1.0, 0.0, 1.0, 0.0], device="cuda")
                for group_of, G in (([i % len(GROUPS) for i in range(len(numels))], len(GROUPS)), ([0] * len(numels), 1)):
                    table = group_segments(members, numels, group_of, start, numel, es, WORLD, RANK)
                    segs = comm.group_segments(table, bk.shard // per_vec, G)
                    groups = torch.tensor([r + [0.0, 0.0] for r in GROUPS[:G]], device="cuda")
                    mask = torch.empty(bk.shard, dtype=torch.long, device="cuda")
                    for vec0, nvec, g, _ in table:
                        mask[vec0 * per_vec:(vec0 + nvec) * per_vec] = g

                    def grouped(nb):
                        st, p = bk.state, bk.param
                        if apply_stage:
                            f = comm.fused_clip_apply_sgd_groups if optimizer == "sgd" else comm.fused_clip_apply_adamw_groups
                            f(p, bk.scratch, clip, *st, hp, groups, segs, nblocks=nb)
                        else:
                            f = comm.fused_allreduce_sgd_groups if optimizer == "sgd" else comm.fused_allreduce_adamw_groups
                            f(bk.grad, p, *st, hp, groups, segs, nblocks=nb)

                    def plain(nb, h):
                        st, p = bk.state, bk.param
                        if apply_stage and optimizer == "sgd":
                            comm.fused_clip_apply_sgd(p, bk.scratch, clip, *st, 0.0, 0.0, 0.0, 1.0, nblocks=nb, hp=h)
                        elif apply_stage:
                            comm.fused_clip_apply_adamw(p, bk.scratch, clip, *st, h, nblocks=nb)
                        elif optimizer == "sgd":
                            comm.fused_allreduce_sgd(bk.grad, p, *st, 0.0, 0.0, 0.0, 1.0, nblocks=nb, hp=h)
                        else:
                            comm.fused_allreduce_adamw(bk.grad, p, *st, h, nblocks=nb)

                    for coef in coefs:
                        if coef is not None:
                            clip[2] = coef
                        for nb in NBS:
                            got = bk.run(lambda: grouped(nb))
                            for g in range(G):
                                h = hp.clone()
                                h[lr_i], h[wd_i] = groups[g, 0], groups[g, 1]
                                want = bk.run(lambda: plain(nb, h))
                                sel = mask == g
                                for a, b in zip(got, want):
                                    assert torch.equal(bits(a[sel]), bits(b[sel])), \
                                        f"{optimizer} {dtype} {len(numels)} tensors G={G} group {g} nb={nb} coef={coef}: bits differ"
                                if G == 1:
                                    assert all(torch.equal(bits(a), bits(b)) for a, b in zip(got, want))
                            cases += 1
    assert comm.status() == 0
    stage = "apply (coefficients 0.3/1e-3/1/0/NaN)" if apply_stage else "one-kernel"
    print(f"rank {RANK}: grouped {stage} SGD and AdamW bitwise equal to the ungrouped kernels per group in {cases} runs "
          f"(fp32/bf16, nblocks {NBS}, multicast={comm.has_multicast})", flush=True)
    teardown()


def job_kernel():
    _oracle(False)


def job_apply():
    _oracle(True)


# ------------------------------------------------------------------ the engine against torch.optim with the same groups
STEPS = 5
HYPER = {"sgd": dict(lr=0.05, momentum=0.9, weight_decay=1e-3), "adamw": dict(lr=2e-3, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.05)}


def _groups(model):
    from bagua_net_b200.parallel import no_weight_decay_groups

    head = list(model[-1].parameters())
    nwd = [p for p in no_weight_decay_groups(model)[0]["params"] if all(p is not q for q in head)]
    return [{"params": nwd, "weight_decay": 0.0}, {"params": head, "lr_scale": 4.0}]


def _torch_groups(ref, lr, wd, scale):
    g = _groups(ref)
    g[0]["lr"] = lr
    g[1].update(lr=lr * scale, weight_decay=wd)
    rest = [p for p in ref.parameters() if all(p is not q for gg in g for q in gg["params"])]
    return g + [{"params": rest, "lr": lr, "weight_decay": wd}]


def job_engine():
    from bagua_net_b200.parallel import BnetDDP, SymmComm

    setup()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    comm = SymmComm(512 << 20)
    probe = small_net().cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    cases = 0
    for dtype in (torch.float32, torch.bfloat16):
        tol_total, tol_worst, _ = TOL[dtype]
        for optimizer in ("sgd", "adamw"):
            hyper = HYPER[optimizer]
            for extra in ({}, {"max_grad_norm": 0.05, "accumulation_steps": 2, "ema_decay": 0.5}):
                k = extra.get("accumulation_steps", 1)
                finals = {}
                for graph in (False, True):
                    torch.manual_seed(0)
                    model = small_net().cuda().to(dtype).to(memory_format=torch.channels_last)
                    ref = small_net().cuda().double()
                    ref.load_state_dict({n: t.double() for n, t in model.state_dict().items()})
                    p0 = [p.detach().double().clone() for p in ref.parameters()]
                    eng = BnetDDP(model, bucket_mb=0.05, comm=comm, optimizer=optimizer, param_groups=_groups(model), **hyper,
                                  **extra)
                    assert len(eng.buckets) > 1
                    eng.enable_cuda_graph(graph)
                    lr, wd, scale = hyper["lr"], hyper["weight_decay"], 4.0
                    kw = {"momentum": 0.9} if optimizer == "sgd" else {"betas": (0.9, 0.99), "eps": 1e-8}
                    opt = (torch.optim.SGD if optimizer == "sgd" else torch.optim.AdamW)(_torch_groups(ref, lr, wd, scale), **kw)
                    ema = [p.detach().clone() for p in ref.parameters()]
                    captured = None
                    for step in range(STEPS):
                        if step == 3:              # a schedule and a group change through the device tables
                            lr, scale = 0.5 * lr, 2.0
                            eng.set_lr(lr)
                            eng.set_param_group(1, lr_scale=scale)
                            for g, glr in zip(opt.param_groups, (lr, lr * scale, lr)):
                                g["lr"] = glr
                        xs, ys = global_batch(step)
                        opt.zero_grad()
                        if dtype == torch.float32:
                            torch.nn.functional.cross_entropy(ref(torch.cat(xs).double()), torch.cat(ys)).backward()
                        else:
                            micro_grads(model, probe, ref, xs, ys, k)
                        eng.train_step(xs[RANK].to(dtype).contiguous(memory_format=torch.channels_last), ys[RANK])
                        if graph:
                            captured = captured or eng._graph
                            assert eng._graph is captured, "set_lr / set_param_group re-captured the graph"
                        if "max_grad_norm" in extra:
                            torch.nn.utils.clip_grad_norm_(ref.parameters(), extra["max_grad_norm"])
                        opt.step()
                        with torch.no_grad():
                            for e, p in zip(ema, ref.parameters()):
                                e.copy_(p if step == 0 else torch.lerp(e, p, 0.5))
                    torch.cuda.synchronize()
                    total, worst = rel_updates(eng, model, ref, p0)
                    tag = f"{str(dtype)[6:]} {optimizer} {extra or 'plain'} graph={graph}"
                    assert total < tol_total and worst < tol_worst, f"{tag}: updates differ from torch: {total:.2e} / {worst:.2e}"
                    assert same_on_every_rank(eng.flat_param), f"{tag}: ranks hold different parameters"
                    if "ema_decay" in extra:
                        with eng.ema_parameters():
                            num = sum(float((p.double() - e).norm() ** 2) for p, e in zip(model.parameters(), ema))
                            den = sum(float(e.norm() ** 2) for e in ema)
                        assert (num / den) ** 0.5 < 1e-2, f"{tag}: EMA differs from torch.lerp: {(num / den) ** 0.5:.2e}"
                    assert comm.status() == 0
                    finals[graph] = torch.cat([b.master for b in eng.buckets])
                    print(f"rank {RANK}: {tag}: rel L2 of updates vs float64 torch.optim with the same groups {total:.2e} total, "
                          f"{worst:.2e} worst bucket", flush=True)
                    for h in eng._hooks:
                        h.remove()
                    del eng
                    cases += 1
                d = float((finals[True] - finals[False]).norm() / finals[False].norm())
                assert d <= tol_total / 100, f"eager and graph trajectories differ: {d:.2e}"
    # a checkpoint resumed mid-run is step-exact
    for optimizer in ("sgd", "adamw"):
        def engine():
            torch.manual_seed(0)
            m = small_net().cuda().to(memory_format=torch.channels_last)
            e = BnetDDP(m, bucket_mb=0.05, comm=comm, optimizer=optimizer, param_groups=_groups(m), **HYPER[optimizer])
            e.enable_cuda_graph(True)
            return m, e

        def steps(e, a, b):
            for step in range(a, b):
                if step == 2:
                    e.set_param_group(0, lr_scale=0.5)
                xs, ys = global_batch(step)
                e.train_step(xs[RANK].contiguous(memory_format=torch.channels_last), ys[RANK])
            torch.cuda.synchronize()

        m, e = engine()
        steps(e, 0, 5)
        want = torch.cat([b.master for b in e.buckets]).clone()
        for h in e._hooks:
            h.remove()
        m, e = engine()
        steps(e, 0, 3)
        sd, osd = {k: v.clone() for k, v in m.state_dict().items()}, e.optimizer_state_dict()
        for h in e._hooks:
            h.remove()
        m, e = engine()
        m.load_state_dict(sd)
        e.load_optimizer_state_dict(osd)
        assert e.param_groups[0]["lr_scale"] == 0.5
        steps(e, 3, 5)
        got = torch.cat([b.master for b in e.buckets])
        assert torch.equal(bits(got), bits(want)), f"{optimizer}: the resumed run differs from the uninterrupted one"
        for h in e._hooks:
            h.remove()
    print(f"rank {RANK}: grouped engine ok in {cases} runs of {STEPS} steps (world {WORLD}, {PER_RANK} samples per rank); "
          "checkpoint resume step-exact", flush=True)
    teardown()


JOBS = {k[4:]: v for k, v in globals().items() if k.startswith("job_")}

if __name__ == "__main__":
    JOBS[sys.argv[1]]()

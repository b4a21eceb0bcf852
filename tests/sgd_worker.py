"""Per-rank bodies of the fused SGD GPU tests (launched by tests/test_fused_sgd.py, one process per GPU)."""
from __future__ import annotations

import math
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from adamw_worker import RANK, WORLD, grads_for, same_on_every_rank, setup, teardown  # noqa: E402

U = 2.0 ** -24                 # fp32 unit roundoff
FLOOR = 4 * 2.0 ** -149        # results in the subnormal range round to a multiple of 2^-149
NAN = float("nan")
SENTINEL = 3.0                 # guard value of the buffers the kernels write: any write, NaN included, changes it

# {lr, momentum, weight_decay, grad_scale}: momentum and decay; plain SGD (torch keeps no buffer) with a gradient scale
# of 1/2; a gradient scale that is not a power of two; lr = 0 (the parameters stay, the buffer still moves)
HPS = [(0.1, 0.9, 1e-2, 1.0), (0.05, 0.0, 0.0, 0.5), (0.1, 0.9, 0.0, 1.0 / 3), (0.0, 0.9, 1e-2, 1.0)]
LR_SCHED = [1.0, 1.0, 0.3, 0.3, 0.1]       # the learning rate changes between steps
NBS = (1, 7, 132, 264)
PAD = 16 * WORLD * 8                       # guard elements on both sides (16-byte aligned in both dtypes)


def f32(x):
    """A hyper-parameter as the kernel sees it (rounded to fp32), in double."""
    return float(torch.tensor(x, dtype=torch.float32))


def pers(nb):
    """Per-rank vector counts for a grid of `nb` CTAs of 512 threads (the SGD kernel takes 2 vectors per thread per
    batch): one vector, a few, the 2-vector loop one short of a full round (tail only after it), exactly full rounds
    (no tail), one over, and one and a half rounds (the tail loop after the 2-vector loop)."""
    r = 2 * 512 * nb
    return (1, 37, r - 1, r, r + 1, 3 * 512 * nb + 5)


def bits(t):
    return t.reshape(-1).view(torch.uint8)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


# ------------------------------------------------------------------ float64 SGD with an fp32 error bound
class Reference:
    """float64 torch.optim.SGD on the kernel's fp32 inputs, over several steps, with the element-wise bound that fp32
    rounding allows (the analysis of csrc/tests/optim_emu_test.cc, errors of earlier steps carried forward):
      B_d = wd B_p + u(wd|p| + k|G|) + F,  B_b' = mu B_b + B_d + u(mu|b| + |d|) + F,  B_p' = B_p + lr B_b' + u(|p| + lr|b'|) + F
    with G = g * coef * gscale, k = 2 for the one-kernel step and 3 for the clipped apply (scratch * coef rounds too).
    Zero hyper-parameters as torch: wd = 0 does not read p, mu = 0 keeps no buffer (b' = d)."""

    def __init__(self, p0: torch.Tensor, b0: torch.Tensor):
        self.p, self.b = p0.double(), b0.double()
        self.bp, self.bb = torch.zeros_like(self.p), torch.zeros_like(self.p)

    def step(self, g: torch.Tensor, lr, mu, wd, gs, coef=None):
        lr, mu, wd, gs = f32(lr), f32(mu), f32(wd), f32(gs)
        k = 2 if coef is None else 3
        G = g.double() * (1.0 if coef is None else f32(coef)) * gs
        d = G if wd == 0 else wd * self.p + G
        b1 = d if mu == 0 else mu * self.b + d
        p1 = self.p - lr * b1
        bd = wd * self.bp + U * (wd * self.p.abs() + k * G.abs()) + FLOOR
        self.bb = mu * self.bb + bd + U * (mu * self.b.abs() + d.abs()) + FLOOR
        self.bp = self.bp + lr * self.bb + U * (self.p.abs() + lr * b1.abs()) + FLOOR
        self.p, self.b = p1, b1

    def worst(self, master, mom):
        """Largest error/bound ratio; inf where the kernel's result is NaN or infinite (the reference is finite here)."""
        r = 0.0
        for got, want, b in ((master, self.p, self.bp), (mom, self.b, self.bb)):
            ratio = ((got.double() - want).abs() / b).nan_to_num(nan=math.inf, posinf=math.inf)
            r = max(r, float(ratio.max()))
        return r


class Buffers:
    """Heap parameters and gradients of up to `nmax` elements and local fp32 master / momentum / scratch shards, each with
    guards of PAD elements on both sides.  `views(n)` hands out the first n elements (shards: n / WORLD).  The buffers
    the kernels write (parameters, master, momentum) get a finite sentinel: an update of a NaN is NaN, so a NaN guard
    would not show a write past the end.  The inputs (gradients, scratch) get NaN: a read past the end makes a result NaN.
    `guards_intact` compares the guards' bits with what was filled in."""

    def __init__(self, comm, nmax, dtype):
        self.pbuf, self.gbuf = comm.alloc(nmax + 2 * PAD, dtype), comm.alloc(nmax + 2 * PAD, dtype)
        smax = nmax // WORLD
        self.mbuf, self.bbuf, self.sbuf = (torch.empty(smax + 2 * PAD, device="cuda") for _ in range(3))

    def views(self, n):
        s = n // WORLD
        for b, v in ((self.pbuf, SENTINEL), (self.gbuf, NAN), (self.mbuf, SENTINEL), (self.bbuf, SENTINEL), (self.sbuf, NAN)):
            b.fill_(v)
        self.filled = [(b[:PAD].clone(), b[PAD + m:].clone()) for b, m in self._guarded(n)]
        return (self.pbuf[PAD:PAD + n], self.gbuf[PAD:PAD + n], self.mbuf[PAD:PAD + s], self.bbuf[PAD:PAD + s],
                self.sbuf[PAD:PAD + s])

    def _guarded(self, n):
        s = n // WORLD
        return ((self.pbuf, n), (self.gbuf, n), (self.mbuf, s), (self.bbuf, s), (self.sbuf, s))

    def guards_intact(self, n):
        return all(same_bits(b[:PAD], lo) and same_bits(b[PAD + m:], hi)
                   for (b, m), (lo, hi) in zip(self._guarded(n), self.filled))


def sync():
    torch.cuda.synchronize()
    if WORLD > 1:
        dist.barrier()


# ------------------------------------------------------------------ the one-kernel step against float64
def job_kernel():
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(512 << 20)
    sizes = sorted({p for nb in NBS for p in pers(nb)})
    worst = {}
    for dtype in (torch.bfloat16, torch.float32):
        E = 16 // torch.tensor([], dtype=dtype).element_size()
        nmax = sizes[-1] * WORLD * E
        bufs = Buffers(comm, nmax, dtype)
        hp = torch.zeros(4, device="cuda")
        # every rank's gradients of every step at the largest size (smaller sizes take a prefix), and their exact sum
        gall = [grads_for(s, nmax, dtype) for s in range(len(LR_SCHED))]
        gsum = [torch.stack([g.double() for g in gs]).sum(0) for gs in gall]
        torch.manual_seed(3)
        p0all = (torch.randn(nmax, device="cuda") * 0.5).to(dtype)
        b0all = torch.randn(nmax // WORLD, device="cuda") * 0.1
        for lr, mu, wd, gs in HPS:
            for per in sizes:
                n = per * WORLD * E
                shard = n // WORLD
                lo, hi = RANK * shard, (RANK + 1) * shard

                def run(nb, use_hp, zero_grads):
                    param, grad, master, mom, _ = bufs.views(n)
                    param.copy_(p0all[:n])
                    master.copy_(param[lo:hi].float())
                    mom.copy_(b0all[:shard])
                    for s, f in enumerate(LR_SCHED):
                        g = gall[s][RANK][:n]
                        grad.copy_(g)
                        hp.copy_(torch.tensor([lr * f, mu, wd, gs]))
                        sync()
                        if use_hp:
                            comm.fused_allreduce_sgd(grad, param, master, mom, 0.5, 0.5, 0.5, 0.5, zero_grads=zero_grads,
                                                     nblocks=nb, hp=hp)
                        else:
                            comm.fused_allreduce_sgd(grad, param, master, mom, lr * f, mu, wd, gs, zero_grads=zero_grads,
                                                     nblocks=nb)
                        torch.cuda.synchronize()
                        tag = f"{dtype} hp={(lr, mu, wd, gs)} per={per} nblocks={nb} hp_entry={use_hp} step {s}"
                        if zero_grads:
                            assert int((grad != 0).sum()) == 0, f"{tag}: gradients were not re-zeroed"
                        else:
                            assert same_bits(grad, g), f"{tag}: gradients changed with zero_grads=False"
                        assert bufs.guards_intact(n), f"{tag}: guard region overwritten"
                    assert same_bits(param[lo:hi], master.to(dtype)), f"{tag}: parameters != master.to(dtype)"
                    assert same_on_every_rank(param), f"{tag}: ranks hold different parameters"
                    return param.clone(), master.clone(), mom.clone()

                got = run(0, True, True)
                ref = Reference(p0all[:n].float()[lo:hi], b0all[:shard])
                for s, f in enumerate(LR_SCHED):
                    ref.step(gsum[s][:n][lo:hi], lr * f, mu, wd, gs)
                w = ref.worst(got[1], got[2])
                worst[dtype] = max(worst.get(dtype, 0.0), w)
                assert w <= 1.0, f"{dtype} hp={(lr, mu, wd, gs)} per={per}: outside the fp32 bound of float64 SGD ({w:.3f})"
                for nb in NBS:
                    if per not in pers(nb):
                        continue
                    for use_hp in (True, False):     # the scalar entry point leaves the gradients in place
                        other = run(nb, use_hp, use_hp)
                        for a, b, what in zip(got, other, ("param", "master", "momentum")):
                            assert same_bits(a, b), \
                                f"{dtype} hp={(lr, mu, wd, gs)} per={per}: nblocks={nb} hp_entry={use_hp} changes {what}"
    assert comm.status() == 0
    print(f"rank {RANK}: fused sgd kernel vs float64: worst error/bound bf16 {worst[torch.bfloat16]:.3f}, "
          f"f32 {worst[torch.float32]:.3f} over {len(HPS)} hyper-parameter sets x {len(sizes)} sizes x 5 steps; bitwise "
          f"equal for nblocks 1/7/132/264 and the scalar / hp entry points (multicast={comm.has_multicast})", flush=True)
    teardown()


# ------------------------------------------------------------------ NaN / Inf gradients against torch.optim.SGD
def job_nonfinite():
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(256 << 20)
    lr = 0.1
    for dtype in (torch.bfloat16, torch.float32):
        n = 8 * WORLD * 4099
        shard = n // WORLD
        lo, hi = RANK * shard, (RANK + 1) * shard
        param, grad = comm.alloc(n, dtype), comm.alloc(n, dtype)
        torch.manual_seed(7)
        p0 = (torch.randn(n, device="cuda") * 0.5).to(dtype)
        idx = torch.arange(0, n, 37, device="cuda")
        vals = torch.tensor([NAN, math.inf, -math.inf], device="cuda").repeat(len(idx) // 3 + 1)[:len(idx)]
        for mu, wd in ((0.9, 1e-2), (0.9, 0.0), (0.0, 1e-2), (0.0, 0.0)):
            param.copy_(p0)
            master = param[lo:hi].float().contiguous()
            mom = torch.zeros_like(master)
            tp = torch.nn.Parameter(p0.float().clone())
            opt = torch.optim.SGD([tp], lr=lr, momentum=mu, weight_decay=wd)
            for s in range(3):
                gs = [g.clone() for g in grads_for(s, n, dtype)]
                if s == 0:
                    for g in gs:                      # every rank puts the specials at the same elements
                        g[idx] = vals.to(dtype)
                grad.copy_(gs[RANK])
                sync()
                comm.fused_allreduce_sgd(grad, param, master, mom, lr, mu, wd)
                torch.cuda.synchronize()
                tp.grad = torch.stack([g.float() for g in gs]).sum(0) / WORLD
                opt.step()
            checks = [("master", master, tp.detach())]
            if mu != 0:                               # torch keeps a momentum buffer only with momentum != 0
                checks.append(("momentum", mom, opt.state[tp]["momentum_buffer"]))
            for name, a, b in checks:
                b = b[lo:hi]
                tag = f"{dtype} momentum={mu} weight_decay={wd}: {name}"
                assert torch.equal(a.isnan(), b.isnan()), \
                    f"{tag}: NaN pattern differs from torch ({int(a.isnan().sum())} NaN, torch {int(b.isnan().sum())})"
                assert torch.equal(a.isinf(), b.isinf()), \
                    f"{tag}: Inf pattern differs from torch ({int(a.isinf().sum())} Inf, torch {int(b.isinf().sum())})"
                assert torch.equal(a[b.isinf()], b[b.isinf()]), f"{tag}: the signs of the infinities differ from torch"
            assert int((master.isnan() | master.isinf()).sum()) == len(idx[(idx >= lo) & (idx < hi)])
            mine, ok = param[lo:hi], ~master.isnan()
            assert torch.equal(mine.isnan(), master.isnan()) and same_bits(mine[ok], master[ok].to(dtype)), \
                "parameters != master.to(dtype)"
            assert same_on_every_rank(param), "ranks hold different parameters"
    assert comm.status() == 0
    print(f"rank {RANK}: fused sgd NaN/+-Inf gradients then finite steps: NaN and Inf patterns = torch.optim.SGD for "
          f"(momentum, weight_decay) in (0.9, 1e-2), (0.9, 0), (0, 1e-2), (0, 0)", flush=True)
    teardown()


# ------------------------------------------------------------------ stage 3 of the clipped step against float64
def job_clip_apply():
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(512 << 20)
    sizes = sorted({p for nb in NBS for p in pers(nb)})
    coefs = (0.3, 1e-3, 1.0, 0.0)
    steps = 3
    worst = {}
    for dtype in (torch.bfloat16, torch.float32):
        E = 16 // torch.tensor([], dtype=dtype).element_size()
        nmax = sizes[-1] * WORLD * E
        bufs = Buffers(comm, nmax, dtype)
        hp = torch.zeros(4, device="cuda")
        clip = torch.zeros(4, device="cuda")
        gen = torch.Generator(device="cuda").manual_seed(50 + RANK)
        sall = [torch.randn(nmax // WORLD, device="cuda", generator=gen) for _ in range(steps)]
        torch.manual_seed(4)
        p0all = (torch.randn(nmax, device="cuda") * 0.5).to(dtype)
        b0all = torch.randn(nmax // WORLD, device="cuda") * 0.1
        for hi_, (lr, mu, wd, gs) in enumerate(HPS):
            # every hyper-parameter set meets every coefficient at a few sizes; all sizes run with one coefficient each
            for si, per in enumerate(sizes):
                coef = coefs[(si + hi_) % len(coefs)]
                n = per * WORLD * E
                shard = n // WORLD
                lo, hi = RANK * shard, (RANK + 1) * shard

                def run(nb, use_hp):
                    c = coef
                    param, _, master, mom, scratch = bufs.views(n)
                    param.copy_(p0all[:n])
                    master.copy_(param[lo:hi].float())
                    mom.copy_(b0all[:shard])
                    clip.copy_(torch.tensor([1.0, 2.0, c, 0.0]))
                    for s in range(steps):
                        scratch.copy_(sall[s][:shard])
                        hp.copy_(torch.tensor([lr * LR_SCHED[s], mu, wd, gs]))
                        sync()
                        if use_hp:
                            comm.fused_clip_apply_sgd(param, scratch, clip, master, mom, 0.5, 0.5, 0.5, 0.5, nblocks=nb, hp=hp)
                        else:
                            comm.fused_clip_apply_sgd(param, scratch, clip, master, mom, lr * LR_SCHED[s], mu, wd, gs,
                                                      nblocks=nb)
                        torch.cuda.synchronize()
                        tag = f"{dtype} hp={(lr, mu, wd, gs)} coef={c} per={per} nblocks={nb} hp_entry={use_hp} step {s}"
                        assert same_bits(scratch, sall[s][:shard]), f"{tag}: the scratch was written"
                        assert bufs.guards_intact(n), f"{tag}: guard region overwritten"
                    assert same_bits(param[lo:hi], master.to(dtype)), f"{tag}: parameters != master.to(dtype)"
                    assert same_on_every_rank(param), f"{tag}: ranks hold different parameters"
                    return param.clone(), master.clone(), mom.clone()

                got = run(0, True)
                ref = Reference(p0all[:n].float()[lo:hi], b0all[:shard])
                for s in range(steps):
                    ref.step(sall[s][:shard], lr * LR_SCHED[s], mu, wd, gs, coef=coef)
                w = ref.worst(got[1], got[2])
                worst[dtype] = max(worst.get(dtype, 0.0), w)
                assert w <= 1.0, f"{dtype} hp={(lr, mu, wd, gs)} coef={coef} per={per}: outside the fp32 bound ({w:.3f})"
                for nb in NBS:
                    if per not in pers(nb):
                        continue
                    for use_hp in (True, False):
                        other = run(nb, use_hp)
                        for a, b, what in zip(got, other, ("param", "master", "momentum")):
                            assert same_bits(a, b), \
                                f"{dtype} hp={(lr, mu, wd, gs)} coef={coef} per={per}: nblocks={nb} hp_entry={use_hp} changes {what}"
        # a NaN coefficient (clip_grad_norm_ of a NaN norm) makes every element NaN
        for lr, mu, wd, gs in HPS:
            per = pers(7)[-1]
            n = per * WORLD * E
            shard = n // WORLD
            lo, hi = RANK * shard, (RANK + 1) * shard
            param, _, master, mom, scratch = bufs.views(n)
            param.copy_(p0all[:n])
            master.copy_(param[lo:hi].float())
            mom.copy_(b0all[:shard])
            scratch.copy_(sall[0][:shard])
            clip.copy_(torch.tensor([1.0, NAN, NAN, 0.0]))
            sync()
            comm.fused_clip_apply_sgd(param, scratch, clip, master, mom, lr, mu, wd, gs)
            torch.cuda.synchronize()
            for name, t in (("master", master), ("momentum", mom), ("param", param)):
                assert bool(t.isnan().all()), f"{dtype} hp={(lr, mu, wd, gs)}: NaN coefficient left {name} partly finite"
            assert bufs.guards_intact(n), "guard region overwritten"
    assert comm.status() == 0
    print(f"rank {RANK}: clipped sgd apply vs float64: worst error/bound bf16 {worst[torch.bfloat16]:.3f}, "
          f"f32 {worst[torch.float32]:.3f} (coefficients {coefs}); bitwise equal for nblocks 1/7/132/264 and the scalar / "
          f"hp entry points; scratch untouched; NaN coefficient gives NaN (multicast={comm.has_multicast})", flush=True)
    teardown()


# ------------------------------------------------------------------ the engine against torch.optim.SGD
KW = dict(width_div=8, fc_dim=128, image_size=32, num_classes=10, dropout=0.0)
LR, WD = 0.05, 1e-2


def batch(step):
    xs, ys = [], []
    for r in range(WORLD):
        torch.manual_seed(1000 + 10 * step + r)
        xs.append(torch.randn(4, 3, 32, 32, device="cuda"))
        ys.append(torch.randint(0, 10, (4,), device="cuda"))
    return torch.cat(xs), torch.cat(ys), xs[RANK].contiguous(memory_format=torch.channels_last), ys[RANK]


def lr_at(step):
    return LR * (0.5 if step >= 4 else 1.0)        # a schedule change after step 4


def make_engine(graph, momentum, max_norm, model=None):
    from bagua_net_b200.models import build_model
    from bagua_net_b200.parallel import BnetDDP

    if model is None:
        torch.manual_seed(0)
        model = build_model("vgg16", **KW).cuda()
    model = model.to(memory_format=torch.channels_last)
    eng = BnetDDP(model, lr=LR, momentum=momentum, weight_decay=WD, bucket_mb=0.25, optimizer="sgd",
                  max_grad_norm=max_norm)
    eng.enable_cuda_graph(graph)
    return model, eng


def engine_step(eng, step, thr):
    _, _, xr, yr = batch(step)
    eng.set_lr(lr_at(step))
    if thr is not None and thr != eng.max_grad_norm:
        eng.set_max_grad_norm(thr)
    eng.train_step(xr, yr)


def job_engine():
    from bagua_net_b200.models import build_model

    setup()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    # thresholds from the step-0 gradient norm (the same for every run): clipped, clipped, far above, then tighter
    torch.manual_seed(0)
    probe = build_model("vgg16", **KW).cuda()
    x, y, _, _ = batch(0)
    torch.nn.functional.cross_entropy(probe(x), y).backward()
    n0 = float(torch.nn.utils.clip_grad_norm_(probe.parameters(), math.inf))
    clipped = [0.5 * n0, 0.5 * n0, 10 * n0, 0.25 * n0, 0.25 * n0, 0.25 * n0]
    # (graph, momentum, thresholds per step or None for the one-kernel step)
    runs = [(False, 0.9, clipped), (True, 0.9, clipped), (False, 0.9, None), (True, 0.9, None), (False, 0.0, clipped)]
    for graph, mu, thresholds in runs:
        tag = f"graph={graph} momentum={mu} clip={thresholds is not None}"
        torch.manual_seed(0)
        ref = build_model("vgg16", **KW).cuda()
        model, eng = make_engine(graph, mu, None if thresholds is None else thresholds[0])
        assert len(eng.buckets) > 1
        opt = torch.optim.SGD(ref.parameters(), lr=LR, momentum=mu, weight_decay=WD)
        p0 = [p.detach().clone() for p in ref.parameters()]
        g, coefs, worst_norm, snap = None, [], 0.0, None
        for step in range(6):
            thr = None if thresholds is None else thresholds[step]
            x, y, _, _ = batch(step)
            if thr is not None:                       # torch's norm of the engine's own parameters at this step
                probe.load_state_dict(model.state_dict())
                probe.zero_grad()
                torch.nn.functional.cross_entropy(probe(x), y).backward()
                want = float(torch.nn.utils.clip_grad_norm_(probe.parameters(), math.inf))
            engine_step(eng, step, thr)
            if graph:
                g = g or eng._graph
                assert eng._graph is g, f"{tag}: the graph was re-captured"
            if thr is not None:
                assert same_on_every_rank(bits(eng.last_grad_norm)), f"{tag}: ranks see different norms"
                got = float(eng.last_grad_norm)
                worst_norm = max(worst_norm, abs(got - want) / want)
                assert abs(got - want) <= 1e-5 * want, (tag, step, got, want)
                coefs.append(float(eng._clip[2]))
            for grp in opt.param_groups:
                grp["lr"] = lr_at(step)
            opt.zero_grad()
            torch.nn.functional.cross_entropy(ref(x), y).backward()
            if thr is not None:
                torch.nn.utils.clip_grad_norm_(ref.parameters(), thr)
            opt.step()
            if step == 2:
                torch.cuda.synchronize()
                snap = ({k: v.clone() for k, v in model.state_dict().items()}, eng.optimizer_state_dict())
        if thresholds is not None:
            assert min(coefs) < 1.0 and coefs[2] == 1.0, (tag, coefs)
        torch.cuda.synchronize()
        num, den, worst = 0.0, 0.0, 0.0
        for a, b, s in zip(model.parameters(), ref.parameters(), p0):
            du, dr = (a.detach().double() - s.double()), (b.detach().double() - s.double())
            e, r = float((du - dr).norm()), float(dr.norm())
            num, den = num + e * e, den + r * r
            worst = max(worst, e / r if r > 0 else (0.0 if e == 0 else float("inf")))
        total = (num / den) ** 0.5
        assert total < 1e-3 and worst < 1e-2, f"{tag}: updates differ from torch SGD: total {total:.2e}, worst {worst:.2e}"
        assert same_on_every_rank(eng.flat_param), f"{tag}: ranks hold different parameters"
        # checkpoint after step 3, resumed into a fresh engine: the same bits at step 6
        torch.manual_seed(0)
        fresh = build_model("vgg16", **KW).cuda()
        fresh.load_state_dict(snap[0])
        fm, fe = make_engine(graph, mu, None if thresholds is None else thresholds[3], fresh)
        fe.load_optimizer_state_dict(snap[1])
        for step in range(3, 6):
            engine_step(fe, step, None if thresholds is None else thresholds[step])
        torch.cuda.synchronize()
        assert torch.equal(fe.flat_param, eng.flat_param), f"{tag}: resumed run differs from the uninterrupted one"
        for b1, b2 in zip(fe.buckets, eng.buckets):
            for t1, t2 in zip(fe._state(b1), eng._state(b2)):
                assert torch.equal(t1, t2), f"{tag}: resumed optimizer state differs"
        assert eng.comm.status() == 0
        extra = (f"; norm vs torch worst rel {worst_norm:.1e}; coefficients {[round(c, 4) for c in coefs]}"
                 if thresholds is not None else "")
        print(f"rank {RANK}: sgd engine ({tag}) vs torch SGD: rel L2 of updates {total:.2e} total, {worst:.2e} worst "
              f"tensor; resume from step 3 bit-identical{extra}", flush=True)
        del eng, fe
    teardown()


JOBS = {k[4:]: v for k, v in globals().items() if k.startswith("job_")}

if __name__ == "__main__":
    JOBS[sys.argv[1]]()

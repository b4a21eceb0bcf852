"""Per-rank bodies of the gradient-clipping GPU tests (launched by tests/test_grad_clip.py, one process per GPU)."""
from __future__ import annotations

import math
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from adamw_worker import RANK, WORLD, same_on_every_rank, setup, teardown  # noqa: E402

from bagua_net_b200.parallel.comm import CLIP_ROW  # noqa: E402

U32 = 2.0 ** -24
U64 = 2.0 ** -53
NAN = float("nan")


def rank_grads(seed, n, dtype, scale=1.0):
    """Every rank's gradient: Gaussian, rounded to `dtype`."""
    out = []
    for r in range(WORLD):
        gen = torch.Generator(device="cuda").manual_seed(seed * 100 + r)
        out.append((torch.randn(n, device="cuda", generator=gen) * scale).to(dtype))
    return out


def guarded(numel, dtype, pad, heap=None):
    """(buffer, inner view): `pad` NaN elements on both sides of `numel`."""
    buf = heap.alloc(numel + 2 * pad, dtype) if heap is not None else torch.empty(numel + 2 * pad, device="cuda", dtype=dtype)
    return buf, buf[pad:pad + numel]


def same_bits_on_every_rank(t: torch.Tensor) -> bool:
    """adamw_worker.same_on_every_rank for a tensor of any shape, 0-dim included (a byte view needs >= 1 dim).  The
    reshape runs on one GPU as well, where the comparison itself returns early."""
    return same_on_every_rank(t.reshape(-1).view(torch.uint8))


def guards_nan(buf, pad):
    return bool(buf[:pad].isnan().all() and buf[-pad:].isnan().all())


# ------------------------------------------------------------------ stage 1 against float64
def job_kernel():
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(256 << 20)
    pad = 16 * WORLD * 8
    worst = 0.0
    for dtype in (torch.bfloat16, torch.float32):
        udt = 2.0 ** -8 if dtype == torch.bfloat16 else U32
        for vec in (4099, 37, 132 * 512 * 2 + 5):
            n = 8 * WORLD * vec
            shard = n // WORLD
            gbuf, grad = guarded(n, dtype, pad, comm)
            sbuf, scratch = guarded(shard, torch.float32, 64)
            pbuf, partial = guarded(CLIP_ROW, torch.float64, 2)
            gs = rank_grads(vec, n, dtype)
            lo, hi = RANK * shard, (RANK + 1) * shard

            def run(nb):
                for b in (gbuf, sbuf, pbuf):
                    b.fill_(NAN)
                grad.copy_(gs[RANK])
                torch.cuda.synchronize()
                if WORLD > 1:
                    dist.barrier()
                comm.fused_clip_reduce_norm(grad, scratch, partial, nblocks=nb)
                torch.cuda.synchronize()
                assert guards_nan(gbuf, pad) and guards_nan(sbuf, 64) and guards_nan(pbuf, 2), "guard region overwritten"
                assert int((grad != 0).sum()) == 0, "gradients were not re-zeroed"
                return scratch.clone(), partial.clone()

            exact = torch.stack([g.double() for g in gs]).sum(0)[lo:hi]
            absum = torch.stack([g.double().abs() for g in gs]).sum(0)[lo:hi]
            for nb in (1, 7, 132, 264):
                s, p = run(nb)
                if WORLD == 1:
                    assert torch.equal(s, gs[0].float()), f"{dtype}: scratch != the upcast gradient"
                else:
                    bound = (WORLD - 1) * U32 * absum + udt * exact.abs()
                    err = (s.double() - exact).abs()
                    assert bool((err <= bound).all()), f"{dtype}: scratch outside the reduction bound"
                assert not p.isnan().any() and bool((p[nb:] == 0).all()), "partial slots beyond the grid not zeroed"
                ref = (s.double() ** 2).sum()
                r = float((p.sum() - ref).abs() / (2 * (shard + 2 * CLIP_ROW) * U64 * ref))
                worst = max(worst, r)
                assert r <= 1.0, f"{dtype}: sum of squares outside its bound ({r:.3f})"
                s2, p2 = run(nb)
                assert torch.equal(s.view(torch.int32), s2.view(torch.int32)) and torch.equal(p.view(torch.int64), p2.view(torch.int64)), \
                    f"{dtype}: nblocks={nb}: a repeat gives different bits"
    assert comm.status() == 0
    print(f"rank {RANK}: clip stage 1 ok: scratch = reduced gradient, sum of squares worst error/bound {worst:.2e}, "
          f"bits repeat for nblocks 1/7/132/264 (multicast={comm.has_multicast})", flush=True)
    teardown()


# ------------------------------------------------------------------ stage 2: norm, coefficient, non-finite gradients
def job_coef():
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(64 << 20)
    n = 8 * WORLD * 1001
    shard = n // WORLD
    lo, hi = RANK * shard, (RANK + 1) * shard
    lr, mu, wd = 0.1, 0.9, 0.01
    pad = 16 * WORLD * 8
    pbuf, param = guarded(n, torch.float32, pad, comm)
    grad = comm.alloc(n, torch.float32)
    scratch = torch.empty(shard, device="cuda")
    partials = torch.full((2, CLIP_ROW), NAN, device="cuda", dtype=torch.float64)
    xchg = comm.alloc(WORLD, torch.float64)
    clip = torch.zeros(4, device="cuda")
    torch.manual_seed(3)
    p0 = torch.randn(n, device="cuda")

    def step(gs, max_norm):
        """The three stages on one bucket; the second partial row stands for a bucket without gradients (zeros)."""
        pbuf.fill_(NAN)
        param.copy_(p0)
        master, mom = param[lo:hi].clone(), torch.zeros(shard, device="cuda")
        grad.copy_(gs[RANK])
        clip[0] = max_norm
        partials[1].zero_()
        torch.cuda.synchronize()
        if WORLD > 1:
            dist.barrier()
        comm.fused_clip_reduce_norm(grad, scratch, partials[0])
        comm.fused_clip_coef(partials, xchg, clip)
        comm.fused_clip_apply_sgd(param, scratch, clip, master, mom, lr, mu, wd)
        torch.cuda.synchronize()
        assert guards_nan(pbuf, pad), "parameter guard overwritten"
        return float(clip[1]), float(clip[2]), param.clone(), master

    def torch_ref(gs, max_norm):
        tp = torch.nn.Parameter(p0.clone())
        tp.grad = torch.stack(gs).sum(0) / WORLD
        norm = torch.nn.utils.clip_grad_norm_([tp], max_norm)
        torch.optim.SGD([tp], lr=lr, momentum=mu, weight_decay=wd).step()
        return float(norm), tp.detach()

    gs = rank_grads(1, n, torch.float32)
    mean = torch.stack([g.double() for g in gs]).sum(0) / WORLD
    exact = float(mean.norm())
    tn, _, _, _ = step(gs, math.inf)
    assert abs(tn - exact) <= 2 * U32 * exact, (tn, exact)
    for max_norm in (0.5 * tn, tn, 2 * tn, math.inf):            # above, at and below the threshold, and never
        t, c, p, master = step(gs, max_norm)
        # (at the threshold the coefficient is tn / (tn + 1e-6) in fp32: 1 or just below it, whatever torch gives)
        want_c = float(torch.clamp(torch.tensor(max_norm, dtype=torch.float32) / (torch.tensor(t) + 1e-6), max=1.0))
        assert t == tn and c == want_c, (max_norm, t, c, want_c)
        if max_norm != tn:
            assert (c < 1.0) == (max_norm < tn), (max_norm, tn, c)
        norm, tp = torch_ref(gs, max_norm)
        assert abs(norm - t) <= 1e-5 * t
        assert torch.allclose(master, tp[lo:hi], rtol=1e-6, atol=1e-6), float((master - tp[lo:hi]).abs().max())
        assert same_on_every_rank(p), "ranks hold different parameters"
    zero = [torch.zeros(n, device="cuda") for _ in range(WORLD)]
    t, c, _, _ = step(zero, 1.0)
    assert t == 0.0 and c == 1.0, (t, c)
    # non-finite gradient elements: the NaN / Inf pattern of clip_grad_norm_ + SGD
    idx = torch.arange(5, n, 97, device="cuda")
    for name, vals in (("nan", [NAN]), ("+inf", [math.inf]), ("-inf", [-math.inf]), ("mixed", [NAN, math.inf, -math.inf])):
        bad = [g.clone() for g in gs]
        v = torch.tensor(vals, device="cuda").repeat(len(idx) // len(vals) + 1)[:len(idx)]
        bad[0][idx] = v                                           # on rank 0 only: the sum carries it to every rank
        t, c, p, master = step(bad, 1.0)
        norm, tp = torch_ref(bad, 1.0)
        assert (t != t) == (norm != norm) and (t == math.inf) == (norm == math.inf), (name, t, norm)
        ref = tp[lo:hi]
        assert torch.equal(master.isnan(), ref.isnan()) and torch.equal(master.isinf(), ref.isinf()), \
            f"{name}: NaN/Inf pattern differs from torch"
    assert comm.status() == 0
    print(f"rank {RANK}: clip coefficient ok: norm {tn:.6g} vs float64 {exact:.6g}; below/at/above/inf thresholds and "
          f"NaN/+-Inf patterns match torch", flush=True)
    teardown()


# ------------------------------------------------------------------ max_norm = inf: bitwise the one-kernel step
def job_identity():
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(256 << 20)
    sizes = [8 * WORLD * 4099, 8 * WORLD * 77]
    lr, mu, wd = 0.05, 0.9, 1e-3
    pad = 16 * WORLD * 8
    cases = 0
    for dtype in (torch.bfloat16, torch.float32):
        pbufs, params = zip(*(guarded(n, dtype, pad, comm) for n in sizes))
        grads = [comm.alloc(n, dtype) for n in sizes]
        gin = [torch.empty(n, device="cuda", dtype=dtype) for n in sizes]
        scratch = [torch.empty(n // WORLD, device="cuda") for n in sizes]
        partials = torch.zeros(len(sizes), CLIP_ROW, device="cuda", dtype=torch.float64)
        xchg = comm.alloc(WORLD, torch.float64)
        clip = torch.tensor([math.inf, 0.0, 0.0, 0.0], device="cuda")
        torch.manual_seed(11)
        p0 = [(torch.randn(n, device="cuda") * 0.1).to(dtype) for n in sizes]
        for kind in ("sgd", "sgd_hp", "adamw"):
            for graph in (False, True):
                results = []
                for clipped in (False, True):
                    for b, p, q in zip(pbufs, params, p0):
                        b.fill_(NAN)
                        p.copy_(q)
                    for g in grads:
                        g.zero_()
                    shard = [p[RANK * (p.numel() // WORLD):(RANK + 1) * (p.numel() // WORLD)] for p in params]
                    nst = 3 if kind == "adamw" else 2
                    state = [(s.float().contiguous(),) + tuple(torch.zeros(s.numel(), device="cuda") for _ in range(nst - 1))
                             for s in shard]
                    hp = (torch.tensor([lr, 0.9, 0.999, 1e-8, 0.01, 1.0 / WORLD, 0.0, 0.0], device="cuda") if kind == "adamw"
                          else torch.tensor([lr, mu, wd, 1.0 / WORLD], device="cuda"))

                    def body():
                        for g, x in zip(grads, gin):
                            g.copy_(x)
                        for k in range(len(sizes)):
                            if clipped:
                                comm.fused_clip_reduce_norm(grads[k], scratch[k], partials[k])
                            elif kind == "adamw":
                                comm.fused_allreduce_adamw(grads[k], params[k], *state[k], hp)
                            else:
                                comm.fused_allreduce_sgd(grads[k], params[k], *state[k], lr, mu, wd,
                                                         hp=hp if kind == "sgd_hp" else None)
                        if clipped:
                            comm.fused_clip_coef(partials, xchg, clip)
                            for k in range(len(sizes)):
                                if kind == "adamw":
                                    comm.fused_clip_apply_adamw(params[k], scratch[k], clip, *state[k], hp)
                                else:
                                    comm.fused_clip_apply_sgd(params[k], scratch[k], clip, *state[k], lr, mu, wd,
                                                              hp=hp if kind == "sgd_hp" else None)
                        if kind == "adamw":
                            hp[6:7].add_(1.0)

                    torch.cuda.synchronize()
                    if WORLD > 1:
                        dist.barrier()
                    g_obj = None
                    if graph:
                        g_obj = torch.cuda.CUDAGraph()
                        with torch.cuda.graph(g_obj):
                            body()
                    for s in range(5):
                        for k, n in enumerate(sizes):
                            gin[k].copy_(rank_grads(1000 * s + k, n, dtype)[RANK])
                        torch.cuda.synchronize()
                        if WORLD > 1:
                            dist.barrier()
                        g_obj.replay() if graph else body()
                    torch.cuda.synchronize()
                    assert all(guards_nan(b, pad) for b in pbufs), f"{dtype} {kind} clipped={clipped}: parameter guard overwritten"
                    results.append(([p.clone() for p in params], [[t.clone() for t in st] for st in state]))
                    del g_obj
                (pa, sa), (pb, sb) = results
                for a, b in zip(pa, pb):
                    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f"{dtype} {kind} graph={graph}: parameters differ"
                for sta, stb in zip(sa, sb):
                    for a, b in zip(sta, stb):
                        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"{dtype} {kind} graph={graph}: state differs"
                assert float(clip[2]) == 1.0 and math.isfinite(float(clip[1]))
                cases += 1
    assert comm.status() == 0
    print(f"rank {RANK}: max_norm=inf is bitwise the one-kernel step in {cases} cases (sgd, sgd_hp, adamw x bf16, f32 x "
          f"eager, graph), 5 steps each", flush=True)
    teardown()


# ------------------------------------------------------------------ stage 1 under staggered CTAs
def job_staggered():
    """The CTA-paired gradient zeroing of stage 1: 64 CTAs on a side stream under a concurrent GEMM, integer gradients,
    so the scratch must hold the exact sum."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(512 << 20)
    n = 8 * WORLD * (64 * 512 * 5 + 4099)
    dtype = torch.bfloat16
    grad = comm.alloc(n, dtype)
    shard = n // WORLD
    scratch = torch.empty(shard, device="cuda")
    partial = torch.empty(CLIP_ROW, device="cuda", dtype=torch.float64)
    side = torch.cuda.Stream()
    a = torch.randn(8192, 8192, device="cuda", dtype=torch.bfloat16)
    for step in range(6):
        grad.copy_(((torch.arange(n, device="cuda") * 3 + RANK + step) % 5 - 2).to(dtype))
        scratch.fill_(NAN)
        torch.cuda.synchronize()
        if WORLD > 1:
            dist.barrier()
        for _ in range(3):
            a @ a
        with torch.cuda.stream(side):
            comm.fused_clip_reduce_norm(grad, scratch, partial, nblocks=64, stream=side)
        torch.cuda.synchronize()
        want = sum(((torch.arange(n, device="cuda") * 3 + r + step) % 5 - 2).float() for r in range(WORLD))
        bad = int((scratch != want[RANK * shard:(RANK + 1) * shard]).sum())
        assert bad == 0, f"rank {RANK} step {step}: {bad} wrong elements (staggered CTAs corrupted the reduction)"
        assert float(partial.sum()) == float((want[RANK * shard:(RANK + 1) * shard].double() ** 2).sum())
        assert int((grad != 0).sum()) == 0, "gradients were not re-zeroed"
    assert comm.status() == 0
    print(f"rank {RANK}: clip stage 1 with 64 staggered CTAs under a concurrent GEMM ok (world {WORLD})", flush=True)
    teardown()


# ------------------------------------------------------------------ the engine against AdamW + clip_grad_norm_
KW = dict(width_div=8, fc_dim=128, image_size=32, num_classes=10, dropout=0.0)
HYPER = dict(lr=2e-3, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.05)


def batch(step):
    xs, ys = [], []
    for r in range(WORLD):
        torch.manual_seed(1000 + 10 * step + r)
        xs.append(torch.randn(4, 3, 32, 32, device="cuda"))
        ys.append(torch.randint(0, 10, (4,), device="cuda"))
    return torch.cat(xs), torch.cat(ys), xs[RANK].contiguous(memory_format=torch.channels_last), ys[RANK]


def job_engine():
    from bagua_net_b200.models import build_model
    from bagua_net_b200.parallel import BnetDDP

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
    thresholds = [0.5 * n0, 0.5 * n0, 10 * n0, 0.25 * n0, 0.25 * n0, 0.25 * n0]
    for graph in (False, True):
        torch.manual_seed(0)
        ref = build_model("vgg16", **KW).cuda()
        torch.manual_seed(0)
        model = build_model("vgg16", **KW).cuda().to(memory_format=torch.channels_last)
        eng = BnetDDP(model, bucket_mb=0.25, optimizer="adamw", max_grad_norm=thresholds[0], **HYPER)
        eng.enable_cuda_graph(graph)
        assert len(eng.buckets) > 1
        opt = torch.optim.AdamW(ref.parameters(), **HYPER)
        p0 = [p.detach().clone() for p in ref.parameters()]
        g, coefs, worst_norm = None, [], 0.0
        for step, thr in enumerate(thresholds):
            x, y, xr, yr = batch(step)
            # torch's norm of the engine's own parameters at this step
            probe.load_state_dict(model.state_dict())
            probe.zero_grad()
            torch.nn.functional.cross_entropy(probe(x), y).backward()
            want = float(torch.nn.utils.clip_grad_norm_(probe.parameters(), math.inf))
            if thr != eng.max_grad_norm:
                eng.set_max_grad_norm(thr)
            eng.train_step(xr, yr)
            if graph:
                g = g or eng._graph
                assert eng._graph is g, "the graph was re-captured"
            got = float(eng.last_grad_norm)
            worst_norm = max(worst_norm, abs(got - want) / want)
            assert abs(got - want) <= 1e-5 * want, (step, got, want)
            assert same_bits_on_every_rank(eng.last_grad_norm), "ranks see different norms"
            coefs.append(float(eng._clip[2]))
            opt.zero_grad()
            torch.nn.functional.cross_entropy(ref(x), y).backward()
            torch.nn.utils.clip_grad_norm_(ref.parameters(), thr)
            opt.step()
        assert min(coefs) < 1.0 and coefs[2] == 1.0, coefs
        torch.cuda.synchronize()
        num, den, worst = 0.0, 0.0, 0.0
        for a, b, s in zip(model.parameters(), ref.parameters(), p0):
            du, dr = (a.detach().double() - s.double()), (b.detach().double() - s.double())
            e, r = float((du - dr).norm()), float(dr.norm())
            num, den = num + e * e, den + r * r
            worst = max(worst, e / r if r > 0 else (0.0 if e == 0 else float("inf")))
        total = (num / den) ** 0.5
        assert total < 1e-3 and worst < 1e-2, f"graph={graph}: updates differ from torch: total {total:.2e}, worst {worst:.2e}"
        assert same_on_every_rank(eng.flat_param), "ranks hold different parameters"
        assert eng.comm.status() == 0
        print(f"rank {RANK}: clipped AdamW engine (graph={graph}) vs torch AdamW + clip_grad_norm_: rel L2 of updates "
              f"{total:.2e} total, {worst:.2e} worst tensor; norm vs torch worst rel {worst_norm:.1e}; coefficients "
              f"{[round(c, 4) for c in coefs]}", flush=True)
        del eng
    teardown()


JOBS = {k[4:]: v for k, v in globals().items() if k.startswith("job_")}

if __name__ == "__main__":
    JOBS[sys.argv[1]]()

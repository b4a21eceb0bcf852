"""Per-rank bodies of the LARS GPU tests (launched by tests/test_fused_lars.py, one process per GPU)."""
from __future__ import annotations

import math
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from adamw_worker import RANK, WORLD, same_on_every_rank, setup, teardown  # noqa: E402
from grad_accum_worker import PER_RANK, TOL, global_batch, micro_grads, rel_updates, small_net  # noqa: E402
from grad_clip_worker import guarded, guards_nan  # noqa: E402

from bagua_net_b200.parallel.comm import LARS_CHUNK  # noqa: E402
from bagua_net_b200.parallel.ddp import lars_segments, plan_buckets  # noqa: E402

U32 = 2.0 ** -24
U64 = 2.0 ** -53
NAN = float("nan")
# tensor sizes with the odd cases: one element, less than a vector, one vector, a tensor over two chunks plus a tail
NUMELS = [1, 7, 8, 9, 1728, 5, 1000, 2 * LARS_CHUNK * 8 + 3, 17, 4096, 3, 64]


def bits(t):
    return t.contiguous().view(torch.uint8)


# ------------------------------------------------------------------ the norm pass against float64
def job_norm():
    """Per chunk slot the sums of squares of master and scratch against float64, for the tables of every rank of world-2
    and world-8 layouts (the kernel is rank-local), NaN guards around every buffer, the same bits for 1, 7 and 264 CTAs
    and on a repeat."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(64 << 20)
    worst, cases = 0.0, 0
    for dtype in (torch.bfloat16, torch.float32):
        es = torch.empty((), dtype=dtype).element_size()
        per_vec = 16 // es
        for lw in (2, 8):
            plan, _ = plan_buckets(NUMELS, es, lw, 64.0)
            start, numel, members = plan[0]
            shard = numel // lw
            for r in range(lw):
                table = lars_segments(members, NUMELS, start, numel, es, lw, r)
                segs = comm.lars_segments(table, shard // per_vec, len(NUMELS))
                nslots = comm._lars_tables[segs.data_ptr()][3]
                mbuf, master = guarded(shard, torch.float32, 64)
                sbuf, scratch = guarded(shard, torch.float32, 64)
                obuf, slots = guarded(2 * nslots, torch.float64, 4)
                slots = slots.view(nslots, 2)
                g = torch.Generator(device="cuda").manual_seed(100 * lw + r + 7 * RANK)
                m0 = torch.randn(shard, device="cuda", generator=g) * 0.1
                s0 = torch.randn(shard, device="cuda", generator=g) * 1e-3

                def run(nb):
                    for b in (mbuf, sbuf, obuf):
                        b.fill_(NAN)
                    master.copy_(m0)
                    scratch.copy_(s0)
                    comm.fused_lars_norm(master, scratch, segs, slots, dtype, nblocks=nb)
                    torch.cuda.synchronize()
                    assert guards_nan(mbuf, 64) and guards_nan(sbuf, 64) and guards_nan(obuf, 4), "guard region overwritten"
                    assert torch.equal(master, m0) and torch.equal(scratch, s0), "the norm pass wrote its inputs"
                    return slots.clone()

                ref = torch.empty(nslots, 2, dtype=torch.float64, device="cuda")
                count = torch.empty(nslots, dtype=torch.float64, device="cuda")
                for vec0, nvec, _, slot0 in table:
                    for c in range((nvec + LARS_CHUNK - 1) // LARS_CHUNK):
                        a, b = (vec0 + c * LARS_CHUNK) * per_vec, (vec0 + min(nvec, (c + 1) * LARS_CHUNK)) * per_vec
                        ref[slot0 + c, 0] = (m0[a:b].double() ** 2).sum()
                        ref[slot0 + c, 1] = (s0[a:b].double() ** 2).sum()
                        count[slot0 + c] = b - a
                first = None
                for nb in (1, 7, 264):
                    got = run(nb)
                    assert not got.isnan().any(), "a slot was not written"
                    bound = 2 * (count[:, None] + 1024) * U64 * ref
                    err = (got - ref).abs()
                    assert bool((err <= bound).all()), f"{dtype} world {lw} rank {r}: slots outside the float64 bound"
                    worst = max(worst, float((err / bound.clamp_min(1e-300)).max()))
                    assert torch.equal(bits(got), bits(run(nb))), "a repeat gives different bits"
                    first = got if first is None else first
                    assert torch.equal(bits(got), bits(first)), f"nblocks={nb}: other bits"
                cases += 1
    assert comm.status() == 0
    print(f"rank {RANK}: LARS norm ok in {cases} tables (world-2 and world-8 layouts, bf16 and f32): worst error/bound "
          f"{worst:.2e}, bits repeat for nblocks 1/7/264", flush=True)
    teardown()


# ------------------------------------------------------------------ the trust kernel
def trust_ref(w2, g2, excluded, hp, coef):
    """The trust ratio and scalars in float64 from the kernel's fp32 inputs, with Apex's special cases."""
    f = lambda v: float(torch.tensor(v, dtype=torch.float32))  # noqa: E731
    lr, mu, wd, gs, eta, eps = (f(v) for v in hp[:6])
    wn, gn = f(math.sqrt(w2)), f(math.sqrt(g2) * gs * coef)
    if excluded or wn == 0 or gn == 0:
        return 1.0, f(gs * coef), 0.0
    if math.isnan(wn) or math.isnan(gn):
        return NAN, NAN, NAN
    t = eta * wn / (gn + wd * wn + eps) if not math.isinf(gn) else 0.0
    return t, f(gs * coef) * t, wd * t


def job_trust():
    """Exclusion, zero norms, NaN and +-Inf sums, the clip coefficient folded in; the sums over the ranks in rank order and
    the same bits of t on every rank."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(64 << 20)
    T = 40
    inf = math.inf
    # per tensor: (w^2, g^2) of rank 0 (the other ranks add (w^2, g^2) * (rank + 1) / 7 on finite entries), excluded
    special = [(4.0, 1e-4, 1), (0.0, 1e-4, 0), (4.0, 0.0, 0), (NAN, 1e-4, 0), (4.0, NAN, 0), (4.0, inf, 0), (inf, 1e-4, 0),
               (0.0, 0.0, 0), (0.0, 0.0, 1), (NAN, NAN, 1)]
    g = torch.Generator().manual_seed(11)
    rows = special + [(float(torch.rand(1, generator=g)) * 10 ** float(torch.randint(-3, 4, (1,), generator=g)),
                       float(torch.rand(1, generator=g)) * 10 ** float(torch.randint(-8, 0, (1,), generator=g)),
                       int(torch.rand(1, generator=g) < 0.2)) for _ in range(T - len(special))]
    hp = torch.tensor([0.1, 0.9, 5e-4, 1.0 / WORLD, 0.001, 1e-8, 0.0, 0.0], device="cuda")
    # two slots per tensor (the second is the rest of the rank's share), so the per-tensor slot sums are exercised
    slots = torch.zeros(2 * T, 2, dtype=torch.float64, device="cuda")
    tables = [[2 * j, 2, e, 0] for j, (_, _, e) in enumerate(rows)]
    tens = comm.lars_tensors(tables, 2 * T)
    xchg = comm.alloc(2 * WORLD * T, torch.float64)
    clip = torch.tensor([1.0, 0.0, 1.0, 0.0], device="cuda")
    scal = torch.full((T, 2), NAN, device="cuda")
    trust = torch.full((T,), NAN, device="cuda")

    def share(v, r):
        return v * (r + 1) / 7 if math.isfinite(v) else v

    for j, (w2, g2, _) in enumerate(rows):
        w, gg = share(w2, RANK), share(g2, RANK)
        slots[2 * j] = torch.tensor([w * 0.25, gg * 0.25])
        slots[2 * j + 1] = torch.tensor([w - w * 0.25 if math.isfinite(w) else 0.0, gg - gg * 0.25 if math.isfinite(gg) else 0.0])
    worst = 0.0
    for coef in (1.0, 0.3, 1e-3, 0.0, NAN):
        clip[2] = coef
        torch.cuda.synchronize()
        if WORLD > 1:
            dist.barrier()
        comm.fused_lars_trust(slots, tens, xchg, clip, hp, scal, trust)
        torch.cuda.synchronize()
        assert same_on_every_rank(trust) and same_on_every_rank(scal), "ranks see different trust ratios"
        c32 = float(torch.tensor(coef, dtype=torch.float32))
        for j, (w2, g2, e) in enumerate(rows):
            tw = sum(share(w2, r) for r in range(WORLD)) if math.isfinite(w2) else w2
            tg = sum(share(g2, r) for r in range(WORLD)) if math.isfinite(g2) else g2
            want = trust_ref(tw, tg, e, hp.tolist(), c32)
            got = (float(trust[j]), float(scal[j, 0]), float(scal[j, 1]))
            for a, b in zip(got, want):
                if math.isnan(b) or math.isinf(b) or b == 0 or a == 1.0 == b:
                    assert (math.isnan(a) and math.isnan(b)) or a == b, (coef, j, rows[j], got, want)
                else:
                    assert abs(a - b) <= 8 * U32 * abs(b), (coef, j, rows[j], got, want)
                    worst = max(worst, abs(a - b) / (8 * U32 * abs(b)))
        assert float(trust[0]) == 1.0 and float(scal[0, 1]) == 0.0                   # excluded
        assert float(trust[1]) == 1.0                                                 # zero weight norm
        if coef == coef:              # (a NaN coefficient makes even a zero gradient's norm NaN, as clip_grad_norm_ does)
            assert float(trust[2]) == 1.0 and float(scal[2, 1]) == 0.0                # zero gradient norm
        if coef == coef and coef > 0:
            assert math.isnan(float(trust[3])) and math.isnan(float(trust[4])) and float(trust[5]) == 0.0
    assert comm.status() == 0
    print(f"rank {RANK}: LARS trust ok: exclusion, zero norms, NaN/Inf, clip coefficients 1/0.3/1e-3/0/NaN, worst "
          f"error/bound {worst:.3f}, same bits on every rank (world {WORLD})", flush=True)
    teardown()


# ------------------------------------------------------------------ the apply stage against float64 per-tensor SGD
def job_apply():
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(256 << 20)
    worst, cases = 0.0, 0
    hp = torch.tensor([0.1, 0.9, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0], device="cuda")
    lr, mu = float(hp[0]), float(hp[1])                                  # (as the kernel sees them, in fp32)
    for dtype in (torch.bfloat16, torch.float32):
        es = torch.empty((), dtype=dtype).element_size()
        per_vec = 16 // es
        # the layouts: the odd tensors, and loop tails around 2 * 512 * nblocks vectors per shard
        for numels in (NUMELS, [per_vec * (2 * 512 * 132 * WORLD) - 8 * per_vec, 8], [per_vec * (2 * 512 * 7 * WORLD + 1), 3]):
            plan, _ = plan_buckets(numels, es, WORLD, 1e9)
            start, numel, members = plan[0]
            shard = numel // WORLD
            table = lars_segments(members, numels, start, numel, es, WORLD, RANK)
            segs = comm.lars_segments(table, shard // per_vec, len(numels))
            pad = 16 * WORLD * 8
            pbuf, param = guarded(numel, dtype, pad, comm)
            sbuf, scratch = guarded(shard, torch.float32, 64)
            mbuf, master = guarded(shard, torch.float32, 64)
            bbuf, mom = guarded(shard, torch.float32, 64)
            g = torch.Generator(device="cuda").manual_seed(17 + RANK + len(numels))
            s0 = torch.randn(shard, device="cuda", generator=g) * 1e-2
            m0 = torch.randn(shard, device="cuda", generator=g)
            b0 = torch.randn(shard, device="cuda", generator=g) * 1e-2
            T = len(numels)
            scal = torch.stack([torch.rand(T, device="cuda", generator=g) * 0.2, torch.rand(T, device="cuda", generator=g) * 1e-3], 1)
            scal[::3, 1] = 0.0                                           # excluded tensors: no weight decay
            sentinel = 1024.0                                            # (exact in bf16)

            def run(nb):
                pbuf.fill_(sentinel)
                for b in (mbuf, bbuf):
                    b.fill_(sentinel)
                sbuf.fill_(NAN)
                scratch.copy_(s0)
                master.copy_(m0)
                mom.copy_(b0)
                torch.cuda.synchronize()
                if WORLD > 1:
                    dist.barrier()
                comm.fused_lars_apply(param, scratch, segs, scal, hp, master, mom, nblocks=nb)
                torch.cuda.synchronize()
                for b, p in ((pbuf, pad), (mbuf, 64), (bbuf, 64)):
                    assert bool((b[:p] == sentinel).all() and (b[-p:] == sentinel).all()), "guard region overwritten"
                assert guards_nan(sbuf, 64)
                return master.clone(), mom.clone(), param.clone()

            # float64 reference per tensor: d = s * gs + wd * p; buf = mu * buf + d; p -= lr * buf
            gs = torch.empty(shard, dtype=torch.float64, device="cuda")
            wd = torch.empty(shard, dtype=torch.float64, device="cuda")
            for vec0, nvec, tensor, _ in table:
                a, b = vec0 * per_vec, (vec0 + nvec) * per_vec
                gs[a:b], wd[a:b] = float(scal[tensor, 0]), float(scal[tensor, 1])
            d = s0.double() * gs + wd * m0.double()
            buf = mu * b0.double() + d
            p = m0.double() - lr * buf
            mag = mu * b0.double().abs() + (s0.double() * gs).abs() + (wd * m0.double()).abs()
            bound_b = 3 * U32 * mag
            bound_p = U32 * (m0.double().abs() + p.abs()) + lr * (bound_b + U32 * buf.abs())
            first = None
            for nb in (1, 7, 132, 264):
                mm, bb, pp = run(nb)
                eb, ep = (bb.double() - buf).abs(), (mm.double() - p).abs()
                assert bool((eb <= bound_b).all() and (ep <= bound_p).all()), f"{dtype} {len(numels)} tensors nblocks={nb}: outside the bound"
                worst = max(worst, float((eb / bound_b.clamp_min(1e-300)).max()), float((ep / bound_p.clamp_min(1e-300)).max()))
                assert torch.equal(pp[RANK * shard:(RANK + 1) * shard], mm.to(dtype)), "parameters are not the rounded masters"
                assert same_on_every_rank(pp), "ranks hold different parameters"
                first = (mm, bb) if first is None else first
                assert torch.equal(bits(mm), bits(first[0])) and torch.equal(bits(bb), bits(first[1])), f"nblocks={nb}: other bits"
                cases += 1
    assert comm.status() == 0
    print(f"rank {RANK}: LARS apply ok in {cases} runs: worst error/bound {worst:.3f}, same bits for nblocks 1/7/132/264 "
          f"(multicast={comm.has_multicast})", flush=True)
    teardown()


# ------------------------------------------------------------------ the engine against float64 LARC + SGD
STEPS = 5
LARS = dict(lr=0.5, momentum=0.9, weight_decay=5e-4, trust_coefficient=0.02, eps=1e-8)


def larc_step(params, opt):
    """NVIDIA Apex LARC(clip=False) on the .grad of the float64 `params`, then `opt` (torch.optim.SGD, no weight decay);
    returns every tensor's trust ratio."""
    ts = []
    with torch.no_grad():
        for p in params:
            t = 1.0
            if p.dim() > 1:
                wn, gn = p.norm(), p.grad.norm()
                if wn != 0 and gn != 0:
                    t = LARS["trust_coefficient"] * wn / (gn + wn * LARS["weight_decay"] + LARS["eps"])
                    p.grad.add_(p, alpha=LARS["weight_decay"]).mul_(t)
                    t = float(t)
            ts.append(t)
    opt.step()
    return ts


def job_engine():
    from bagua_net_b200.parallel import BnetDDP, SymmComm

    setup()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    comm = SymmComm(256 << 20)
    torch.manual_seed(0)
    probe = small_net().cuda().double()
    xs, ys = global_batch(0)
    torch.nn.functional.cross_entropy(probe(torch.cat(xs).double()), torch.cat(ys)).backward()
    n0 = float(torch.nn.utils.clip_grad_norm_(probe.parameters(), math.inf))
    thresholds = [0.5 * n0, 10 * n0, 0.25 * n0, 0.5 * n0, 0.25 * n0]
    probe = small_net().cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    cases = 0
    for dtype in (torch.float32, torch.bfloat16):
        tol_total, tol_worst, tol_norm = TOL[dtype]
        for k in (1, 2):
            for clipped in (False, True):
                finals = {}
                for graph in (False, True):
                    torch.manual_seed(0)
                    model = small_net().cuda().to(dtype).to(memory_format=torch.channels_last)
                    ref = small_net().cuda().double()
                    ref.load_state_dict({n: t.double() for n, t in model.state_dict().items()})
                    p0 = [p.detach().double().clone() for p in ref.parameters()]
                    eng = BnetDDP(model, bucket_mb=0.05, comm=comm, optimizer="lars", accumulation_steps=k,
                                  max_grad_norm=thresholds[0] if clipped else None, **LARS)
                    assert len(eng.buckets) > 1
                    eng.enable_cuda_graph(graph)
                    opt = torch.optim.SGD(ref.parameters(), lr=LARS["lr"], momentum=LARS["momentum"])
                    worst_t = 0.0
                    for step in range(STEPS):
                        xs, ys = global_batch(step)
                        thr = thresholds[step] if clipped else math.inf
                        if clipped and thr != eng.max_grad_norm:
                            eng.set_max_grad_norm(thr)
                        if step == 3:                                   # a schedule change through the device block
                            eng.set_lr(0.5 * LARS["lr"])
                            for g in opt.param_groups:
                                g["lr"] = 0.5 * LARS["lr"]
                        opt.zero_grad()
                        if dtype == torch.float32:
                            torch.nn.functional.cross_entropy(ref(torch.cat(xs).double()), torch.cat(ys)).backward()
                        else:
                            micro_grads(model, probe, ref, xs, ys, k)
                        x = xs[RANK].to(dtype).contiguous(memory_format=torch.channels_last)
                        eng.train_step(x, ys[RANK])
                        want_norm = float(torch.nn.utils.clip_grad_norm_(ref.parameters(), thr))
                        want_t = larc_step(list(ref.parameters()), opt)
                        got_t = eng.last_trust_ratios.tolist()
                        assert same_on_every_rank(eng.last_trust_ratios), "ranks see different trust ratios"
                        for a, b in zip(got_t, want_t):
                            worst_t = max(worst_t, abs(a - b) / b)
                        assert worst_t <= 100 * tol_norm, (dtype, k, clipped, graph, step, worst_t)
                        if clipped:
                            got = float(eng.last_grad_norm)
                            assert abs(got - want_norm) <= tol_norm * want_norm, (dtype, k, graph, step, got, want_norm)
                    torch.cuda.synchronize()
                    assert float(eng.flat_grad.abs().max()) == 0.0, "gradients left behind"
                    total, worst = rel_updates(eng, model, ref, p0)
                    tag = f"{str(dtype)[6:]} k={k} clipped={clipped} graph={graph}"
                    assert total < tol_total and worst < tol_worst, f"{tag}: updates differ from LARC + SGD: total {total:.2e}, worst {worst:.2e}"
                    assert same_on_every_rank(eng.flat_param), f"{tag}: ranks hold different parameters"
                    assert comm.status() == 0
                    finals[graph] = torch.cat([b.master for b in eng.buckets])
                    print(f"rank {RANK}: {tag}: rel L2 of updates vs float64 LARC + SGD {total:.2e} total, {worst:.2e} worst "
                          f"bucket; trust ratios worst rel {worst_t:.1e}", flush=True)
                    for h in eng._hooks:
                        h.remove()
                    del eng
                    cases += 1
                d = float((finals[True] - finals[False]).norm() / finals[False].norm())
                assert d <= tol_total / 100, f"eager and graph trajectories differ: {d:.2e}"
    print(f"rank {RANK}: LARS engine ok in {cases} runs of {STEPS} steps (world {WORLD}, {PER_RANK} samples per rank)", flush=True)
    teardown()


JOBS = {k[4:]: v for k, v in globals().items() if k.startswith("job_")}

if __name__ == "__main__":
    JOBS[sys.argv[1]]()

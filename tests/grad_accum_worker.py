"""Per-rank bodies of the gradient-accumulation GPU tests (launched by tests/test_grad_accum.py, one process per GPU)."""
from __future__ import annotations

import math
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from adamw_worker import RANK, WORLD, same_on_every_rank, setup, teardown  # noqa: E402
from grad_clip_worker import guarded, guards_nan, rank_grads, same_bits_on_every_rank  # noqa: E402

from bagua_net_b200.parallel.comm import CLIP_ROW  # noqa: E402

U32 = 2.0 ** -24
U64 = 2.0 ** -53
NAN = float("nan")


# ------------------------------------------------------------------ the accumulating stage 1 against float64
def job_kernel():
    """scratch + sum over ranks of grad, in fp32: against float64, with NaN guards around gradients, scratch and partial
    row, the partial row against the float64 sum of squares of the result, the same bits for 1, 7, 132 and 264 CTAs,
    gradients re-zeroed, and from a zeroed scratch the store-only kernel's result."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(256 << 20)
    pad = 16 * WORLD * 8
    worst_sum, worst_sq = 0.0, 0.0
    for dtype in (torch.bfloat16, torch.float32):
        udt = 2.0 ** -8 if dtype == torch.bfloat16 else U32
        for vec in (4099, 37, 132 * 512 * 2 + 5):
            n = 8 * WORLD * vec
            shard = n // WORLD
            gbuf, grad = guarded(n, dtype, pad, comm)
            sbuf, scratch = guarded(shard, torch.float32, 64)
            pbuf, partial = guarded(CLIP_ROW, torch.float64, 2)
            gs = rank_grads(vec, n, dtype)
            gen = torch.Generator(device="cuda").manual_seed(7 * vec + RANK)
            s0 = torch.randn(shard, device="cuda", generator=gen) * 3.0        # what earlier micro-batches left
            lo, hi = RANK * shard, (RANK + 1) * shard

            def run(nb, start, accumulate=True):
                for b in (gbuf, sbuf, pbuf):
                    b.fill_(NAN)
                scratch.copy_(start)
                grad.copy_(gs[RANK])
                torch.cuda.synchronize()
                if WORLD > 1:
                    dist.barrier()
                (comm.fused_accum_reduce_norm if accumulate else comm.fused_clip_reduce_norm)(grad, scratch, partial, nblocks=nb)
                torch.cuda.synchronize()
                assert guards_nan(gbuf, pad) and guards_nan(sbuf, 64) and guards_nan(pbuf, 2), "guard region overwritten"
                assert int((grad != 0).sum()) == 0, "gradients were not re-zeroed"
                return scratch.clone(), partial.clone()

            gsum = torch.stack([g.double() for g in gs]).sum(0)[lo:hi]
            absum = torch.stack([g.double().abs() for g in gs]).sum(0)[lo:hi]
            exact = s0.double() + gsum
            # the rank sum as the store-only stage bounds it (grad_clip_worker.job_kernel), then one fp32 rounding of the add
            bound_g = (WORLD - 1) * U32 * absum + udt * gsum.abs() if WORLD > 1 else torch.zeros_like(gsum)
            bound = bound_g + U32 * (exact.abs() + bound_g)
            first = None
            for nb in (1, 7, 132, 264):
                s, p = run(nb, s0)
                if WORLD == 1:
                    assert torch.equal(s, s0 + gs[0].float()), f"{dtype}: scratch != scratch + gradient in fp32"
                err = (s.double() - exact).abs()
                assert bool((err <= bound).all()), f"{dtype}: scratch outside the accumulation bound"
                worst_sum = max(worst_sum, float((err / bound.clamp_min(1e-300)).max()))
                assert not p.isnan().any() and bool((p[nb:] == 0).all()), "partial slots beyond the grid not zeroed"
                ref = (s.double() ** 2).sum()                             # over the NEW scratch values
                r = float((p.sum() - ref).abs() / (2 * (shard + 2 * CLIP_ROW) * U64 * ref))
                worst_sq = max(worst_sq, r)
                assert r <= 1.0, f"{dtype}: sum of squares outside its bound ({r:.3f})"
                s2, p2 = run(nb, s0)
                assert torch.equal(s.view(torch.int32), s2.view(torch.int32)) and torch.equal(p.view(torch.int64), p2.view(torch.int64)), \
                    f"{dtype}: nblocks={nb}: a repeat gives different bits"
                if first is None:
                    first = s
                assert torch.equal(s.view(torch.int32), first.view(torch.int32)), f"{dtype}: nblocks={nb}: other scratch bits"
                # from a zeroed scratch: what the store-only stage gives (+-0 aside)
                za, pa = run(nb, torch.zeros_like(s0))
                zc, pc = run(nb, s0, accumulate=False)
                assert torch.equal(za, zc) and torch.equal(pa, pc), f"{dtype}: nblocks={nb}: 0 + g differs from the store"
    assert comm.status() == 0
    print(f"rank {RANK}: accumulating stage 1 ok: scratch + g worst error/bound {worst_sum:.3f}, sum of squares worst "
          f"error/bound {worst_sq:.2e}, bits repeat for nblocks 1/7/132/264, zero start == store "
          f"(multicast={comm.has_multicast})", flush=True)
    teardown()


# ------------------------------------------------------------------ the engine against torch on the global batch
PER_RANK = 8                      # samples per rank and optimizer step (k micro-batches of 8/k)
STEPS = 5
SGD = dict(lr=0.05, momentum=0.9, weight_decay=1e-3)
ADAMW = dict(lr=2e-3, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.05)
# The float64 reference takes one step per optimizer step on the gradient of the mean loss over the GLOBAL batch (every
# rank's samples, all k micro-batches).
# * fp32 (TF32 off): a float64 copy of the model runs the global batch in one pass.  The forward and backward passes agree
#   with float64 to ~1e-6 per gradient, and AdamW's normalisation amplifies that for elements whose gradient is near zero:
#   relative L2 of the updates after STEPS steps below 1e-3 over all parameters and 1e-2 for the worst bucket (the bound
#   of grad_clip_worker's engine job); the reported norm within 1e-4 of torch's.
# * bf16: a float64 pass would differ from the bf16 model by bf16 rounding in every activation, which hides what is
#   tested here.  So the gradient of every micro-batch of every rank is computed by a bf16 copy of the engine's current
#   model (the same kernels on the same bits as the engine's own backward), summed in float64 and divided by world * k.
#   What remains is the engine's fp32 arithmetic -- the rank sum, the accumulation in the fp32 scratch, the update -- a
#   few 2^-24 per element and step; AdamW's normalisation amplifies it where the gradient is near zero, and a master
#   weight on a bf16 rounding boundary may round the other way and change the next gradients by a bf16 ulp: 2^-10 total,
#   2^-6 for the worst bucket, and the norm within 1e-5.
TOL = {torch.float32: (1e-3, 1e-2, 1e-4), torch.bfloat16: (2.0 ** -10, 2.0 ** -6, 1e-5)}


def small_net():
    """No BatchNorm: per-micro-batch statistics would make accumulation differ from the global batch by design."""
    return torch.nn.Sequential(torch.nn.Conv2d(3, 32, 3, padding=1), torch.nn.ReLU(), torch.nn.Conv2d(32, 64, 3, padding=1),
                               torch.nn.ReLU(), torch.nn.AdaptiveAvgPool2d(4), torch.nn.Flatten(), torch.nn.Linear(1024, 128),
                               torch.nn.ReLU(), torch.nn.Linear(128, 10))


def global_batch(step):
    """Every rank's samples of `step` (different on every rank) and the concatenation over ranks."""
    xs, ys = [], []
    for r in range(WORLD):
        g = torch.Generator(device="cuda").manual_seed(5000 + 10 * step + r)
        xs.append(torch.randn(PER_RANK, 3, 16, 16, device="cuda", generator=g))
        ys.append(torch.randint(0, 10, (PER_RANK,), device="cuda", generator=g))
    return xs, ys


def as_masters(eng, model, tensors):
    """`tensors` (one per parameter of `model`, float64) laid out as this rank's fp32 master shards of `eng`, one per
    bucket: the updates are compared on the masters, because a bf16 parameter rounds away updates below its ulp."""
    flat = torch.zeros(eng.flat_param.numel(), dtype=torch.float64, device="cuda")
    base, es = eng.flat_param.data_ptr(), eng.flat_param.element_size()
    for p, t in zip(model.parameters(), tensors):
        flat.as_strided(p.shape, p.stride(), (p.data_ptr() - base) // es).copy_(t)
    out = []
    for b in eng.buckets:
        shard = b.numel // WORLD
        out.append(flat[b.start + RANK * shard:b.start + (RANK + 1) * shard])
    return out


def rel_updates(eng, model, ref, p0):
    """Relative L2 error of the engine's master updates against the reference's, over all and for the worst bucket."""
    num, den, worst = 0.0, 0.0, 0.0
    for b, r1, s in zip(eng.buckets, as_masters(eng, model, [p.detach() for p in ref.parameters()]), as_masters(eng, model, p0)):
        du, dr = b.master.double() - s, r1 - s
        e, r = float((du - dr).norm()), float(dr.norm())
        num, den = num + e * e, den + r * r
        worst = max(worst, e / r if r > 0 else (0.0 if e == 0 else float("inf")))
    return (num / den) ** 0.5, worst


def micro_grads(model, probe, ref, xs, ys, k):
    """bf16 reference gradient: every rank's k micro-batches through a bf16 copy of `model` (its parameters as they are
    before this step), summed in float64 and divided by world * k, into `ref`'s .grad."""
    probe.load_state_dict(model.state_dict())
    total = [torch.zeros_like(p) for p in ref.parameters()]
    for x, y in zip(xs, ys):
        x = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        for xm, ym in zip(x.split(PER_RANK // k), y.split(PER_RANK // k)):
            probe.zero_grad()
            torch.nn.functional.cross_entropy(probe(xm).float(), ym).backward()
            for t, p in zip(total, probe.parameters()):
                t += p.grad.double()
    for t, p in zip(total, ref.parameters()):
        p.grad = t / (WORLD * k)


def job_engine():
    from bagua_net_b200.parallel import BnetDDP, SymmComm

    setup()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    comm = SymmComm(256 << 20)
    # clipping thresholds from the step-0 norm: clipped, far above, clipped harder, ...
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
        for k in (2, 4):
            for optimizer in ("sgd", "adamw"):
                for clipped in (False, True):
                    finals = {}
                    for graph in (False, True):
                        torch.manual_seed(0)
                        model = small_net().cuda().to(dtype).to(memory_format=torch.channels_last)
                        ref = small_net().cuda().double()
                        ref.load_state_dict({n: t.double() for n, t in model.state_dict().items()})
                        p0 = [p.detach().double().clone() for p in ref.parameters()]
                        hyper = ADAMW if optimizer == "adamw" else SGD
                        eng = BnetDDP(model, bucket_mb=0.05, comm=comm, optimizer=optimizer, accumulation_steps=k,
                                      max_grad_norm=thresholds[0] if clipped else None, **hyper)
                        assert len(eng.buckets) > 1
                        eng.enable_cuda_graph(graph)
                        opt = (torch.optim.AdamW if optimizer == "adamw" else torch.optim.SGD)(ref.parameters(), **hyper)
                        worst_norm = 0.0
                        for step in range(STEPS):
                            xs, ys = global_batch(step)
                            thr = thresholds[step] if clipped else math.inf
                            if clipped and thr != eng.max_grad_norm:
                                eng.set_max_grad_norm(thr)
                            if optimizer == "sgd" and step == 3:                 # a schedule change: hp in device memory
                                eng.set_lr(0.5 * SGD["lr"])
                                for g in opt.param_groups:
                                    g["lr"] = 0.5 * SGD["lr"]
                            opt.zero_grad()
                            if dtype == torch.float32:
                                torch.nn.functional.cross_entropy(ref(torch.cat(xs).double()), torch.cat(ys)).backward()
                            else:
                                micro_grads(model, probe, ref, xs, ys, k)
                            x = xs[RANK].to(dtype).contiguous(memory_format=torch.channels_last)
                            eng.train_step(x, ys[RANK])
                            assert eng.micro_step == 0
                            want = float(torch.nn.utils.clip_grad_norm_(ref.parameters(), thr))
                            opt.step()
                            if clipped:
                                got = float(eng.last_grad_norm)
                                worst_norm = max(worst_norm, abs(got - want) / want)
                                assert abs(got - want) <= tol_norm * want, (dtype, k, optimizer, graph, step, got, want)
                                assert same_bits_on_every_rank(eng.last_grad_norm), "ranks see different norms"
                        torch.cuda.synchronize()
                        assert float(eng.flat_grad.abs().max()) == 0.0, "gradients left behind"
                        total, worst = rel_updates(eng, model, ref, p0)
                        tag = f"{str(dtype)[6:]} k={k} {optimizer} clipped={clipped} graph={graph}"
                        assert total < tol_total and worst < tol_worst, f"{tag}: updates differ from torch: total {total:.2e}, worst {worst:.2e}"
                        assert same_on_every_rank(eng.flat_param), f"{tag}: ranks hold different parameters"
                        assert comm.status() == 0
                        finals[graph] = torch.cat([b.master for b in eng.buckets])
                        print(f"rank {RANK}: {tag}: rel L2 of updates vs float64 torch {total:.2e} total, {worst:.2e} worst "
                              f"bucket" + (f"; norm worst rel {worst_norm:.1e}" if clipped else ""), flush=True)
                        for h in eng._hooks:
                            h.remove()
                        del eng
                        cases += 1
                    d = float((finals[True] - finals[False]).norm() / finals[False].norm())
                    assert d <= tol_total / 100, f"eager and graph trajectories differ: {d:.2e}"
                    if d:
                        print(f"rank {RANK}: eager vs graph master weights rel L2 {d:.1e}", flush=True)
    print(f"rank {RANK}: accumulating engine ok in {cases} runs of {STEPS} steps (world {WORLD})", flush=True)
    teardown()


JOBS = {k[4:]: v for k, v in globals().items() if k.startswith("job_")}

if __name__ == "__main__":
    JOBS[sys.argv[1]]()

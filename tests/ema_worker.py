"""Per-rank bodies of the EMA GPU tests (launched by tests/test_ema.py, one process per GPU)."""
from __future__ import annotations

import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from adamw_worker import RANK, WORLD, same_on_every_rank, setup, teardown  # noqa: E402
from grad_accum_worker import ADAMW, PER_RANK, SGD, TOL, as_masters, global_batch, micro_grads, small_net  # noqa: E402
from grad_clip_worker import guarded, guards_nan  # noqa: E402
from lars_worker import LARS, larc_step  # noqa: E402

U32 = 2.0 ** -24
NAN = float("nan")


def bits(t):
    return t.contiguous().view(torch.uint8)


def lerp_f64(e, m, w):
    """torch.lerp's two branches in float64 on the kernel's fp32 inputs (w: the fp32 weight)."""
    e, m = e.double(), m.double()
    d = m - e
    return e + w * d if abs(w) < 0.5 else m - d * (1.0 - w)


# ------------------------------------------------------------------ the kernels against float64
def job_update():
    """bnet_ema_update over shards around the ends of its vector loop for 1, 7, 132 and 264 CTAs, NaN guards around both
    shards: the lerp in both branches against float64 (NaN and +-Inf elements included), the same bits for every grid, the
    copy step bitwise the master, a skipped step touching nothing; bnet_ema_advance over a run of steps."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(64 << 20)
    worst, cases = 0.0, 0
    sizes = sorted({n for nb in (1, 7, 132, 264) for n in (4 * 512 * nb - 1, 4 * 512 * nb, 4 * 512 * nb + 1, 5 * 512 * nb + 3)}
                   | {1, 2, 513})
    for n4 in sizes:
        n = 4 * n4
        mbuf, master = guarded(n, torch.float32, 64)
        ebuf, ema = guarded(n, torch.float32, 64)
        g = torch.Generator(device="cuda").manual_seed(n4 + 31 * RANK)
        m0 = torch.randn(n, device="cuda", generator=g)
        e0 = m0 + torch.randn(n, device="cuda", generator=g) * 1e-2
        if n >= 16:                                   # NaN and +-Inf in either operand
            m0[:6] = torch.tensor([NAN, math.inf, -math.inf, 1.0, 1.0, 1.0])
            e0[:6] = torch.tensor([1.0, 1.0, 1.0, NAN, math.inf, -math.inf])

        def run(blk_vals, nb):
            for b in (mbuf, ebuf):
                b.fill_(NAN)
            master.copy_(m0)
            ema.copy_(e0)
            blk = torch.tensor(blk_vals, dtype=torch.float32, device="cuda")
            comm.ema_update(master, ema, blk, nblocks=nb)
            torch.cuda.synchronize()
            assert guards_nan(mbuf, 64) and guards_nan(ebuf, 64), "guard region overwritten"
            assert torch.equal(bits(master), bits(m0)), "the update wrote the master"
            assert torch.equal(blk.cpu(), torch.tensor(blk_vals, dtype=torch.float32)), "the update wrote the block"
            return ema.clone()

        for w in (0.3, 0.8):
            w32 = float(torch.tensor(w, dtype=torch.float32))
            ref = lerp_f64(e0, m0, w32)
            fin = ref.isfinite()
            bound = (1 + 2.0 ** -13) * U32 * (ref.abs() + min(w32, 1 - w32) * (m0.double() - e0.double()).abs())
            first = None
            for nb in (1, 7, 132, 264):
                got = run([w, 3.0, 5.0, 4.0], nb)                       # step 6 of every 3: an EMA step, not a copy
                err = (got.double() - ref).abs()
                assert bool((err[fin] <= bound[fin]).all()), f"n4={n4} w={w} nblocks={nb}: outside the bound"
                assert torch.equal(got[~fin].isnan(), ref[~fin].isnan()), "NaN pattern differs from torch.lerp's"
                nonnan = ~fin & ~ref.isnan()
                assert torch.equal(got[nonnan].double(), ref[nonnan]), "infinities differ from torch.lerp's"
                if bool(fin.any()):
                    worst = max(worst, float((err[fin] / bound[fin].clamp_min(1e-300)).max()))
                first = got if first is None else first
                assert torch.equal(bits(got), bits(first)), f"nblocks={nb}: other bits"
                cases += 1
        for nb in (1, 264):
            assert torch.equal(bits(run([0.3, 3.0, 2.0, 0.0], nb)), bits(m0)), "the copy step is not the master"   # step 3
            assert torch.equal(bits(run([0.3, 3.0, 3.0, 2.0], nb)), bits(e0)), "a skipped step touched the EMA"    # step 4
            cases += 2
    # the advance kernel over a run of steps, with a reset in the middle
    blk = torch.tensor([0.25, 3.0, 0.0, 0.0], device="cuda")
    step, n_avg = 0, 0
    for s in range(1, 40):
        if s == 20:
            blk[3] = 0.0
            n_avg = 0
        comm.ema_advance(blk)
        n_avg += s % 3 == 0
        step = s
        assert blk.tolist() == [0.25, 3.0, float(step), float(n_avg)], (s, blk.tolist())
    assert comm.status() == 0
    print(f"rank {RANK}: EMA update ok in {cases} runs over {len(sizes)} shard sizes: worst error/bound {worst:.3f}, same bits "
          f"for nblocks 1/7/132/264, copy and skip bitwise; advance ok over 39 steps", flush=True)
    teardown()


# ------------------------------------------------------------------ the engine
STEPS = 6
DECAY = 0.6                 # weight 0.4: the lerp's first branch; set_ema_decay(0.3) at step 3: weight 0.7, its second


def rel_ema(eng, model, avg, p0):
    """Relative L2 error of the engine's EMA shards (minus the start) against the reference EMA's, over all and for the
    worst bucket."""
    num, den, worst = 0.0, 0.0, 0.0
    for b, r1, s in zip(eng.buckets, as_masters(eng, model, [p.detach() for p in avg.module.parameters()]), as_masters(eng, model, p0)):
        du, dr = b.ema.double() - s, r1 - s
        e, r = float((du - dr).norm()), float(dr.norm())
        num, den = num + e * e, den + r * r
        worst = max(worst, e / r if r > 0 else (0.0 if e == 0 else float("inf")))
    return (num / den) ** 0.5, worst


def job_engine():
    from torch.optim.swa_utils import AveragedModel, get_ema_multi_avg_fn

    from bagua_net_b200.parallel import BnetDDP, SymmComm

    setup()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    comm = SymmComm(256 << 20)
    probe = small_net().cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    cases, worst_own = 0, 0.0
    for dtype in (torch.float32, torch.bfloat16):
        tol_total, tol_worst, _ = TOL[dtype]
        for optimizer in ("sgd", "adamw", "lars"):
            hyper = {"sgd": SGD, "adamw": ADAMW, "lars": LARS}[optimizer]
            for every in (1, 2):
                for k in (1, 2):
                    for graph in (False, True):
                        torch.manual_seed(0)
                        model = small_net().cuda().to(dtype).to(memory_format=torch.channels_last)
                        ref = small_net().cuda().double()
                        ref.load_state_dict({n: t.double() for n, t in model.state_dict().items()})
                        p0 = [p.detach().double().clone() for p in ref.parameters()]
                        eng = BnetDDP(model, bucket_mb=0.05, comm=comm, optimizer=optimizer, accumulation_steps=k,
                                      ema_decay=DECAY, ema_every=every, **hyper)
                        assert len(eng.buckets) > 1
                        eng.enable_cuda_graph(graph)
                        if optimizer == "adamw":
                            opt = torch.optim.AdamW(ref.parameters(), **hyper)
                        else:
                            opt = torch.optim.SGD(ref.parameters(), lr=hyper["lr"], momentum=hyper["momentum"],
                                                  weight_decay=0.0 if optimizer == "lars" else hyper["weight_decay"])
                        avg = AveragedModel(ref, multi_avg_fn=get_ema_multi_avg_fn(DECAY), use_buffers=False)
                        own = torch.cat([b.master for b in eng.buckets]).double()   # float64 EMA of the engine's masters
                        bound = torch.zeros_like(own)        # ... and the fp32 bound of the engine's EMA around it
                        n_avg, decay, g0 = 0, DECAY, None
                        tag = f"{str(dtype)[6:]} {optimizer} every={every} k={k} graph={graph}"
                        for step in range(1, STEPS + 1):
                            if step == 3:                    # a decay schedule and a restart, through the device block
                                eng.set_ema_decay(0.3)
                                avg.multi_avg_fn, decay = get_ema_multi_avg_fn(0.3), 0.3
                            if step == 5:
                                eng.reset_ema()
                                avg.n_averaged.fill_(0)
                                n_avg = 0
                            xs, ys = global_batch(step)
                            opt.zero_grad()
                            if dtype == torch.float32:
                                torch.nn.functional.cross_entropy(ref(torch.cat(xs).double()), torch.cat(ys)).backward()
                            else:
                                micro_grads(model, probe, ref, xs, ys, k)
                            eng.train_step(xs[RANK].to(dtype).contiguous(memory_format=torch.channels_last), ys[RANK])
                            if optimizer == "lars":
                                larc_step(list(ref.parameters()), opt)
                            else:
                                opt.step()
                            if graph:
                                g0 = eng._graph if g0 is None else g0
                                assert eng._graph is g0, "the EMA changes re-captured the step"
                            masters = torch.cat([b.master for b in eng.buckets]).double()
                            if step % every == 0:
                                avg.update_parameters(ref)
                                w32 = float(torch.tensor(1.0 - decay, dtype=torch.float32))
                                if n_avg == 0:                       # the copy is exact
                                    own, bound = masters.clone(), torch.zeros_like(own)
                                else:
                                    # the lerp carries the error of the EMA it starts from times 1 - w, and its own two
                                    # roundings add u(|r| + min(w, 1 - w)|master - ema|) (job_update)
                                    d = (masters - own).abs()
                                    own = lerp_f64(own, masters, w32)
                                    bound = (1 - w32) * bound + 1.001 * U32 * (own.abs() + min(w32, 1 - w32) * (d + bound))
                                n_avg += 1
                            got = torch.cat([b.ema for b in eng.buckets]).double()
                            err = (got - own).abs()
                            assert bool((err <= bound).all()), f"{tag} step {step}: EMA outside the fp32 bound of its own masters"
                            worst_own = max(worst_own, float((err / bound.clamp_min(1e-300)).max()))
                            assert bool((err[bound == 0] == 0).all())
                        assert eng._ema.tolist()[2:] == [float(STEPS), float(n_avg)]
                        torch.cuda.synchronize()
                        assert float(eng.flat_grad.abs().max()) == 0.0, "gradients left behind"
                        total, worst = rel_ema(eng, model, avg, p0)
                        assert total < tol_total and worst < tol_worst, f"{tag}: EMA differs from AveragedModel: total {total:.2e}, worst {worst:.2e}"
                        # evaluation on the EMA weights: published on every rank, then the trained parameters back, bitwise
                        before = eng.flat_param.clone()
                        with eng.ema_parameters():
                            for b in eng.buckets:
                                shard = b.numel // WORLD
                                assert torch.equal(bits(b.param[RANK * shard:(RANK + 1) * shard]), bits(b.ema.to(dtype)))
                            assert same_on_every_rank(eng.flat_param), f"{tag}: ranks hold different EMA parameters"
                            model(xs[RANK].to(dtype).contiguous(memory_format=torch.channels_last))
                        torch.cuda.synchronize()
                        assert torch.equal(bits(eng.flat_param), bits(before)), f"{tag}: parameters not restored"
                        assert same_on_every_rank(eng.flat_param)
                        assert comm.status() == 0
                        print(f"rank {RANK}: {tag}: EMA vs float64 AveragedModel rel L2 {total:.2e} total, {worst:.2e} worst "
                              f"bucket", flush=True)
                        for h in eng._hooks:
                            h.remove()
                        del eng
                        cases += 1
    print(f"rank {RANK}: EMA engine ok in {cases} runs of {STEPS} steps (world {WORLD}, {PER_RANK} samples per rank); worst "
          f"error/bound against the float64 EMA of the engine's own masters {worst_own:.3f}", flush=True)
    teardown()


JOBS = {k[4:]: v for k, v in globals().items() if k.startswith("job_")}

if __name__ == "__main__":
    JOBS[sys.argv[1]]()

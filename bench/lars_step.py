#!/usr/bin/env python
"""What LARS costs in the fused data-parallel step, on one GPU.

1. Optimizer time at the real tensor shapes of VGG16 (32 tensors, 138.4 M parameters) and ResNet-50 (161 tensors,
   25.6 M), built on the meta device and laid out in 64 MB buckets of bf16 parameters as BnetDDP lays them out:
   * lars: every stage of the LARS step (per bucket reduce into the fp32 scratch; per bucket the per-chunk norms of
     master and scratch; once the trust kernel; per bucket the update from the scratch with per-tensor scalars);
   * clipped_fused_sgd: the same staging without the per-tensor work (per bucket reduce + sum of squares, once the
     coefficient, per bucket the clipped SGD update);
   * torch_larc_sgd_foreach: LARC in torch foreach ops on fp32 master weights (per-tensor norms, trust ratios,
     weight decay and scaling of the non-excluded tensors), torch.optim.SGD(foreach=True), then the cast back to bf16.
   CUDA events time `--steps` whole steps after `--warmup`; the variants alternate for `--rounds` rounds (median).
   Bytes per bf16 parameter from the algorithm: clipped SGD 30 (stage 1: gradient read 2, scratch written 4, gradient
   zeroed 2; stage 3: scratch read 4, master and momentum read and written 16, parameter written 2); LARS 38 (the norm
   pass reads master and scratch, 8 more); the torch variant is charged 38 as well.
2. End to end: BnetDDP.train_step img/s on ResNet-50, bf16, batch `--batch`, 224 x 224, under a CUDA graph, with
   optimizer="sgd" and optimizer="lars", alternating for `--e2e-rounds` rounds.

  python bench/lars_step.py --out profiles/lars_step
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))      # (`bench` is also bench.py at the root)
from optimizer_step import DATASHEET_HBM_BPS, card  # noqa: E402
from bagua_net_b200.models import build_model  # noqa: E402
from bagua_net_b200.parallel import SymmComm  # noqa: E402
from bagua_net_b200.parallel.comm import CLIP_ROW, LARS_CHUNK  # noqa: E402
from bagua_net_b200.parallel.ddp import lars_segments, plan_buckets  # noqa: E402

BYTES_PER_PARAM = {"clipped_fused_sgd": 30, "lars": 38, "torch_larc_sgd_foreach": 38}
LR, MU, WD, ETA, EPS = 0.1, 0.9, 5e-5, 0.001, 1e-8


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / steps


def shapes(name):
    with torch.device("meta"):
        model = build_model(name)
    return [tuple(p.shape) for p in model.parameters()]


def optimizer_times(args, results):
    for model in ("vgg16", "resnet50"):
        shp = shapes(model)
        numels = [int(torch.Size(s).numel()) for s in shp]
        plan, total = plan_buckets(numels, 2, 1, 64.0)
        comm = SymmComm(2 * total * 2 + (64 << 20))
        flat_p, flat_g = comm.alloc(total, torch.bfloat16), comm.alloc(total, torch.bfloat16)
        flat_p.normal_(0, 0.02)
        flat_g.zero_()
        views = [(flat_g[s:s + n], flat_p[s:s + n]) for s, n, _ in plan]
        master = [p.float() for _, p in views]
        mom = [torch.zeros_like(x) for x in master]
        scratch = [torch.zeros_like(x) for x in master]
        partials = torch.zeros(len(plan), CLIP_ROW, device="cuda", dtype=torch.float64)
        xchg = comm.alloc(2 * len(shp), torch.float64)
        clip = torch.tensor([1.0, 0.0, 0.0, 0.0], device="cuda")
        one = torch.tensor([float("inf"), 0.0, 1.0, 0.0], device="cuda")
        hp = torch.tensor([LR, MU, WD, 1.0, ETA, EPS, 0.0, 0.0], device="cuda")
        # the LARS tables, as the engine builds them
        segs, slots, tensors, base = [], [], [[0, 0, int(len(s) <= 1), 0] for s in shp], 0
        for start, numel, members in plan:
            table = lars_segments(members, numels, start, numel, 2, 1, 0)
            segs.append(comm.lars_segments(table, numel // 8, len(shp)))
            n = sum((v + LARS_CHUNK - 1) // LARS_CHUNK for _, v, _, _ in table)
            for _, v, pi, s0 in table:
                tensors[pi][:2] = [base + s0, (v + LARS_CHUNK - 1) // LARS_CHUNK]
            slots.append((base, base + n))
            base += n
        all_slots = torch.zeros(base, 2, dtype=torch.float64, device="cuda")
        tens = comm.lars_tensors(tensors, base)
        scal = torch.zeros(len(shp), 2, device="cuda")
        trust = torch.ones(len(shp), device="cuda")
        # the torch reference: fp32 master tensors of the real shapes
        tparams = [torch.nn.Parameter(torch.randn(s, device="cuda") * 0.02) for s in shp]
        for t in tparams:
            t.grad = torch.randn_like(t) * 1e-3
        opt = torch.optim.SGD(tparams, lr=LR, momentum=MU, foreach=True)
        big = [t for t in tparams if t.dim() > 1]
        bf16 = [torch.empty(s, device="cuda", dtype=torch.bfloat16) for s in shp]

        def clipped_fused_sgd():
            for k, (g, _) in enumerate(views):
                comm.fused_clip_reduce_norm(g, scratch[k], partials[k])
            comm.fused_clip_coef(partials, xchg, clip, grad_scale=1.0)
            for (_, p), s, a, b in zip(views, scratch, master, mom):
                comm.fused_clip_apply_sgd(p, s, clip, a, b, 0.0, 0.0, 0.0, 1.0, hp=hp)

        def lars():
            for k, (g, _) in enumerate(views):
                comm.fused_clip_reduce_norm(g, scratch[k], partials[k])
            for k, (a, b) in enumerate(slots):
                comm.fused_lars_norm(master[k], scratch[k], segs[k], all_slots[a:b], torch.bfloat16)
            comm.fused_lars_trust(all_slots, tens, xchg, one, hp, scal, trust)
            for k, (_, p) in enumerate(views):
                comm.fused_lars_apply(p, scratch[k], segs[k], scal, hp, master[k], mom[k])

        def torch_larc():
            with torch.no_grad():
                grads = [t.grad for t in big]
                wn = torch.stack(torch._foreach_norm(big))
                gn = torch.stack(torch._foreach_norm(grads))
                t = ETA * wn / (gn + WD * wn + EPS)
                t = torch.where((wn != 0) & (gn != 0), t, torch.ones_like(t))
                torch._foreach_add_(grads, big, alpha=WD)
                torch._foreach_mul_(grads, list(t.unbind()))
            opt.step()
            torch._foreach_copy_(bf16, [p.detach() for p in tparams])

        variants = {"clipped_fused_sgd": clipped_fused_sgd, "lars": lars, "torch_larc_sgd_foreach": torch_larc}
        for fn in variants.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fn in variants.items():
                times[k].append(timed(fn, args.steps))
        n = sum(numels)
        row = {"tensors": len(shp), "params": n, "buckets": len(plan), "norm_slots": base}
        for k, ts in times.items():
            ts = sorted(ts)
            us = ts[len(ts) // 2]
            bps = BYTES_PER_PARAM[k] * n / (us * 1e-6)
            row[k] = {"us_per_step_median": round(us, 1), "us_per_step_min": round(ts[0], 1), "us_per_step_max": round(ts[-1], 1),
                      "achieved_tb_per_s": round(bps / 1e12, 3), "share_of_datasheet_hbm_bw": round(bps / DATASHEET_HBM_BPS, 3)}
        row["lars_minus_clipped_sgd_us"] = round(row["lars"]["us_per_step_median"] - row["clipped_fused_sgd"]["us_per_step_median"], 1)
        row["torch_over_lars_time"] = round(row["torch_larc_sgd_foreach"]["us_per_step_median"] / row["lars"]["us_per_step_median"], 3)
        results["optimizer"][model] = row
        assert comm.status() == 0 and bool(torch.isfinite(trust).all())
        del opt, tparams, master, mom, scratch, views, flat_p, flat_g
        comm.close()
        torch.cuda.empty_cache()


def end_to_end(args, results):
    from bagua_net_b200.parallel import BnetDDP

    x = torch.randn(args.batch, 3, 224, 224, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (args.batch,), device="cuda")
    engines = {}
    for name in ("sgd", "lars"):
        torch.manual_seed(0)
        model = build_model("resnet50").cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
        eng = BnetDDP(model, optimizer=name, lr=LR, momentum=MU, weight_decay=WD, bucket_mb=64.0)
        eng.enable_cuda_graph(True)
        for _ in range(args.warmup):
            eng.train_step(x, y)
        engines[name] = eng
    torch.cuda.synchronize()
    imgs = {k: [] for k in engines}
    for _ in range(args.e2e_rounds):
        for k, eng in engines.items():
            us = timed(lambda: eng.train_step(x, y), args.e2e_steps)
            imgs[k].append(args.batch / (us * 1e-6))
    for k, v in imgs.items():
        v = sorted(v)
        results["end_to_end"][k] = {"img_per_s_median": round(v[len(v) // 2], 1), "img_per_s_min": round(v[0], 1),
                                    "img_per_s_max": round(v[-1], 1)}
    t = engines["lars"].last_trust_ratios
    results["end_to_end"]["lars_trust_ratio_range"] = [float(t.min()), float(t.max())]
    results["end_to_end"]["lars_over_sgd_img_per_s"] = round(
        results["end_to_end"]["lars"]["img_per_s_median"] / results["end_to_end"]["sgd"]["img_per_s_median"], 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/lars_step")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--e2e-steps", type=int, default=30)
    ap.add_argument("--e2e-rounds", type=int, default=5)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lars_step.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    results = {"card": card(), "bucket_mb": 64, "param_dtype": "bf16", "steps_per_window": args.steps, "rounds": args.rounds,
               "bytes_per_param": BYTES_PER_PARAM, "datasheet_hbm_tb_per_s": DATASHEET_HBM_BPS / 1e12, "optimizer": {},
               "end_to_end": {}}
    optimizer_times(args, results)
    if not args.no_e2e:
        end_to_end(args, results)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "lars_step.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(results))


if __name__ == "__main__":
    main()

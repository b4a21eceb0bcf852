#!/usr/bin/env python
"""What gradient clipping by global norm costs in the fused data-parallel step, on one GPU.

1. Optimizer time for VGG16's (138.4 M) and ResNet-50's (25.6 M) parameter counts as bf16 parameters in 64 MB buckets,
   laid out as bench/optimizer_step.py does:
   * fused_adamw: the one-kernel all-reduce + AdamW step per bucket;
   * clipped_fused_adamw: all three stages of the clipped step (per bucket reduce + sum of squares, once the norm and
     the coefficient, per bucket the update from the fp32 scratch);
   * torch_clip_adamw_fused: torch.nn.utils.clip_grad_norm_(foreach=True), torch.optim.AdamW(fused=True) on fp32
     master weights, then the cast back to bf16.
   CUDA events time `--steps` whole steps after `--warmup`; the variants alternate for `--rounds` rounds (median).
   Bytes per bf16 parameter from the algorithm: fused AdamW 30 B, clipped 38 B (stage 1: gradient read 2, scratch
   written 4, gradient zeroed 2; stage 3: scratch read 4, three fp32 states read and written 24, parameter written 2);
   the torch variant is charged 38 B as well.
2. End to end: BnetDDP.train_step img/s on VGG16, bf16, batch 32, 224 x 224, under a CUDA graph, with max_grad_norm
   None and 1.0, alternating for `--e2e-rounds` rounds.

  python bench/grad_clip_step.py --out profiles/grad_clip_step
"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))      # (`bench` is also bench.py at the root)
from optimizer_step import DATASHEET_HBM_BPS, MODELS, buckets, card  # noqa: E402
from bagua_net_b200.parallel import SymmComm  # noqa: E402
from bagua_net_b200.parallel.comm import CLIP_ROW  # noqa: E402

BYTES_PER_PARAM = {"fused_adamw": 30, "clipped_fused_adamw": 38, "torch_clip_adamw_fused": 38}


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / steps


def optimizer_times(args, results):
    total = sum(buckets(MODELS["vgg16"]))
    comm = SymmComm(2 * total * 2 + (64 << 20))
    flat_p, flat_g = comm.alloc(total, torch.bfloat16), comm.alloc(total, torch.bfloat16)
    flat_p.normal_(0, 0.02)
    flat_g.zero_()
    xchg = comm.alloc(1, torch.float64)
    clip = torch.tensor([1.0, 0.0, 0.0, 0.0], device="cuda")
    hp = torch.tensor([1e-4, 0.9, 0.999, 1e-8, 0.01, 1.0, 0.0, 0.0], device="cuda")
    for model, n in MODELS.items():
        sizes = buckets(n)
        views, off = [], 0
        for s in sizes:
            views.append((flat_g[off:off + s], flat_p[off:off + s]))
            off += s
        master = [p.float() for _, p in views]
        m1 = [torch.zeros_like(x) for x in master]
        m2 = [torch.zeros_like(x) for x in master]
        scratch = [torch.zeros_like(x) for x in master]
        partials = torch.zeros(len(sizes), CLIP_ROW, device="cuda", dtype=torch.float64)
        tparams = [torch.nn.Parameter(x.clone()) for x in master]
        for t in tparams:
            t.grad = torch.zeros_like(t)
        opt = torch.optim.AdamW(tparams, lr=1e-4, weight_decay=0.01, fused=True)

        def fused_adamw():
            for (g, p), a, b, c in zip(views, master, m1, m2):
                comm.fused_allreduce_adamw(g, p, a, b, c, hp)

        def clipped_fused_adamw():
            for k, (g, _) in enumerate(views):
                comm.fused_clip_reduce_norm(g, scratch[k], partials[k])
            comm.fused_clip_coef(partials, xchg, clip)
            for (_, p), s, a, b, c in zip(views, scratch, master, m1, m2):
                comm.fused_clip_apply_adamw(p, s, clip, a, b, c, hp)

        def torch_clip_adamw():
            torch.nn.utils.clip_grad_norm_(tparams, 1.0, foreach=True)
            opt.step()
            for (_, p), t in zip(views, tparams):
                p.copy_(t.detach())

        variants = {"fused_adamw": fused_adamw, "clipped_fused_adamw": clipped_fused_adamw,
                    "torch_clip_adamw_fused": torch_clip_adamw}
        for fn in variants.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fn in variants.items():
                times[k].append(timed(fn, args.steps))
        row = {"params": n, "buckets": len(sizes)}
        for k, ts in times.items():
            ts = sorted(ts)
            us = ts[len(ts) // 2]
            bps = BYTES_PER_PARAM[k] * n / (us * 1e-6)
            row[k] = {"us_per_step_median": round(us, 1), "us_per_step_min": round(ts[0], 1), "us_per_step_max": round(ts[-1], 1),
                      "achieved_tb_per_s": round(bps / 1e12, 3), "share_of_datasheet_hbm_bw": round(bps / DATASHEET_HBM_BPS, 3)}
        row["clipped_over_fused_time"] = round(row["clipped_fused_adamw"]["us_per_step_median"] /
                                               row["fused_adamw"]["us_per_step_median"], 3)
        row["torch_over_clipped_time"] = round(row["torch_clip_adamw_fused"]["us_per_step_median"] /
                                               row["clipped_fused_adamw"]["us_per_step_median"], 3)
        results["optimizer"][model] = row
        del opt, tparams, master, m1, m2, scratch
        torch.cuda.empty_cache()
    assert comm.status() == 0 and math.isfinite(float(clip[1]))
    comm.close()


def end_to_end(args, results):
    from bagua_net_b200.models import build_model
    from bagua_net_b200.parallel import BnetDDP

    x = torch.randn(args.batch, 3, 224, 224, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (args.batch,), device="cuda")
    engines = {}
    for name, max_norm in (("max_grad_norm_none", None), ("max_grad_norm_1", 1.0)):
        torch.manual_seed(0)
        model = build_model("vgg16", fused=True).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
        eng = BnetDDP(model, lr=0.01, momentum=0.9, weight_decay=1e-4, bucket_mb=64.0, max_grad_norm=max_norm)
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
    results["end_to_end"]["last_grad_norm"] = float(engines["max_grad_norm_1"].last_grad_norm)
    results["end_to_end"]["clipped_over_unclipped_img_per_s"] = round(
        results["end_to_end"]["max_grad_norm_1"]["img_per_s_median"] / results["end_to_end"]["max_grad_norm_none"]["img_per_s_median"], 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/grad_clip_step")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--e2e-steps", type=int, default=30)
    ap.add_argument("--e2e-rounds", type=int, default=5)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("grad_clip_step.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    results = {"card": card(), "bucket_mb": 64, "param_dtype": "bf16", "steps_per_window": args.steps, "rounds": args.rounds,
               "bytes_per_param": BYTES_PER_PARAM, "datasheet_hbm_tb_per_s": DATASHEET_HBM_BPS / 1e12, "optimizer": {},
               "end_to_end": {}}
    optimizer_times(args, results)
    if not args.no_e2e:
        end_to_end(args, results)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "grad_clip_step.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(results))


if __name__ == "__main__":
    main()

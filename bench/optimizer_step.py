#!/usr/bin/env python
"""Optimizer step time on one GPU: the fused all-reduce + AdamW kernel, the fused all-reduce + SGD kernel, and what a
user would otherwise run for AdamW (torch.optim.AdamW(fused=True) on fp32 master weights, then the cast back to bf16).

The parameter counts are VGG16's (138.4 M) and ResNet-50's (25.6 M), as bf16 parameters in the engine's 64 MB buckets.
Every variant steps over all buckets of a model; CUDA events time `--steps` whole steps after `--warmup` steps, and the
variants alternate for `--rounds` rounds in one process (the median window is reported).

Achieved bandwidth uses the bytes the algorithm has to move per bf16 parameter, not what an implementation happens to
move: AdamW 30 B (gradient read and re-zeroed 4, parameter written 2, three fp32 states read and written 24), SGD 22 B
(4 + 2 + two fp32 states read and written 16).  The torch variant is charged AdamW's 30 B as well (it moves more: fp32
gradients, and a second pass for the cast).  The share of peak is against the H100 SXM data sheet's 3.35 TB/s of HBM3.

  python bench/optimizer_step.py --out profiles/optimizer_step
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bagua_net_b200.parallel import SymmComm  # noqa: E402

MODELS = {"vgg16": 138_357_544, "resnet50": 25_557_032}
BYTES_PER_PARAM = {"fused_adamw": 30, "fused_sgd": 22, "torch_adamw_fused": 30}
DATASHEET_HBM_BPS = 3.35e12
BUCKET_ELEMS = (64 << 20) // 2            # 64 MB of bf16


def card():
    out = {"name": torch.cuda.get_device_name(), "power_limit_w": None, "max_sm_clock_mhz": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        pl, clk = (v.strip() for v in r.stdout.strip().splitlines()[0].split(","))
        out["power_limit_w"], out["max_sm_clock_mhz"] = float(pl), float(clk)
    except Exception as ex:   # noqa: BLE001 - the card's name is still reported
        out["power_limit_error"] = f"{type(ex).__name__}: {ex}"
    return out


def buckets(n):
    sizes, left = [], n
    while left > 0:
        b = min(BUCKET_ELEMS, left)
        sizes.append((b + 63) // 64 * 64)
        left -= b
    return sizes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/optimizer_step")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optimizer_step.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    total = sum(buckets(MODELS["vgg16"]))
    comm = SymmComm(2 * total * 2 + (64 << 20))
    flat_p, flat_g = comm.alloc(total, torch.bfloat16), comm.alloc(total, torch.bfloat16)
    flat_p.normal_(0, 0.02)
    flat_g.zero_()
    hp_adamw = torch.tensor([1e-4, 0.9, 0.999, 1e-8, 0.01, 1.0, 0.0, 0.0], device="cuda")
    hp_sgd = torch.tensor([1e-4, 0.9, 1e-4, 1.0], device="cuda")
    results = {"card": card(), "bucket_mb": 64, "param_dtype": "bf16", "steps_per_window": args.steps,
               "rounds": args.rounds, "datasheet_hbm_tb_per_s": DATASHEET_HBM_BPS / 1e12,
               "bytes_per_param": BYTES_PER_PARAM, "models": {}}
    for model, n in MODELS.items():
        sizes = buckets(n)
        views, off = [], 0
        for s in sizes:
            views.append((flat_g[off:off + s], flat_p[off:off + s]))
            off += s
        master = [p.float() for _, p in views]
        m1 = [torch.zeros_like(x) for x in master]
        m2 = [torch.zeros_like(x) for x in master]
        mom = [torch.zeros_like(x) for x in master]
        # torch: fp32 parameters with fp32 gradients in place already (the gradient cast is not charged to it)
        tparams = [torch.nn.Parameter(x.clone()) for x in master]
        for t in tparams:
            t.grad = torch.zeros_like(t)
        opt = torch.optim.AdamW(tparams, lr=1e-4, weight_decay=0.01, fused=True)

        def fused_adamw():
            for (g, p), a, b, c in zip(views, master, m1, m2):
                comm.fused_allreduce_adamw(g, p, a, b, c, hp_adamw)

        def fused_sgd():
            for (g, p), a, b in zip(views, master, mom):
                comm.fused_allreduce_sgd(g, p, a, b, 0.0, 0.0, 0.0, hp=hp_sgd)

        def torch_adamw():
            opt.step()
            for (_, p), t in zip(views, tparams):
                p.copy_(t.detach())

        variants = {"fused_adamw": fused_adamw, "fused_sgd": fused_sgd, "torch_adamw_fused": torch_adamw}
        for fn in variants.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, fn in variants.items():          # alternate the variants: drift hits them alike
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    fn()
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) * 1e3 / args.steps)
        row = {"params": n, "buckets": len(sizes)}
        for k, ts in times.items():
            ts = sorted(ts)
            us = ts[len(ts) // 2]
            bps = BYTES_PER_PARAM[k] * n / (us * 1e-6)
            row[k] = {"us_per_step_median": round(us, 1), "us_per_step_min": round(ts[0], 1), "us_per_step_max": round(ts[-1], 1),
                      "achieved_tb_per_s": round(bps / 1e12, 3),
                      "share_of_datasheet_hbm_bw": round(bps / DATASHEET_HBM_BPS, 3)}
        row["adamw_over_sgd_time"] = round(row["fused_adamw"]["us_per_step_median"] / row["fused_sgd"]["us_per_step_median"], 3)
        row["torch_over_fused_adamw_time"] = round(row["torch_adamw_fused"]["us_per_step_median"] /
                                                   row["fused_adamw"]["us_per_step_median"], 3)
        results["models"][model] = row
        del opt, tparams, master, m1, m2, mom
        torch.cuda.empty_cache()
    assert comm.status() == 0
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "optimizer_step.json")
    with open(path, "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(results))


if __name__ == "__main__":
    main()

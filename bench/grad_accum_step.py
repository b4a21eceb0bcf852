#!/usr/bin/env python
"""What gradient accumulation costs and saves in the fused data-parallel step, on one GPU.

1. Stage 1 alone, per bucket, for VGG16's parameter count (138.4 M) as bf16 parameters in 64 MB buckets, laid out as
   bench/optimizer_step.py does:
   * store: the stage of a bucket's first micro-batch in a step (fused_clip_reduce_norm): reduce, store the fp32 scratch,
     sum of squares, zero the gradients;
   * accumulate: every later micro-batch's stage (fused_accum_reduce_norm): the same, adding to the scratch.
   CUDA events time `--steps` passes over all buckets after `--warmup`; the two alternate for `--rounds` rounds (median).
   Bytes per bf16 parameter from the algorithm: store 8 B (gradient read 2, scratch written 4, gradient zeroed 2),
   accumulate 12 B (gradient read 2, scratch read 4 and written 4, gradient zeroed 2).
2. End to end: BnetDDP.train_step img/s on VGG16, bf16, `--micro-batch` images per micro-batch, 224 x 224, SGD, under
   a CUDA graph, for accumulation_steps k in `--ks` (a step is k micro-batches), alternating for `--e2e-rounds` rounds.

  python bench/grad_accum_step.py --out profiles/grad_accum_step
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))      # (`bench` is also bench.py at the root)
from optimizer_step import DATASHEET_HBM_BPS, MODELS, buckets, card  # noqa: E402
from bagua_net_b200.parallel import SymmComm  # noqa: E402
from bagua_net_b200.parallel.comm import CLIP_ROW  # noqa: E402

BYTES_PER_PARAM = {"store": 8, "accumulate": 12}


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / steps


def stage1_times(args, results):
    n = MODELS["vgg16"]
    sizes = buckets(n)
    total = sum(sizes)
    comm = SymmComm(total * 2 + (64 << 20))
    flat_g = comm.alloc(total, torch.bfloat16)
    flat_g.normal_(0, 1e-3)
    grads, off = [], 0
    for s in sizes:
        grads.append(flat_g[off:off + s])
        off += s
    scratch = [torch.zeros(s, device="cuda") for s in sizes]
    partials = torch.zeros(len(sizes), CLIP_ROW, device="cuda", dtype=torch.float64)

    def store():
        for k, g in enumerate(grads):
            comm.fused_clip_reduce_norm(g, scratch[k], partials[k])

    def accumulate():
        for k, g in enumerate(grads):
            comm.fused_accum_reduce_norm(g, scratch[k], partials[k])

    variants = {"store": store, "accumulate": accumulate}
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
        row[k] = {"us_per_pass_median": round(us, 1), "us_per_pass_min": round(ts[0], 1), "us_per_pass_max": round(ts[-1], 1),
                  "achieved_tb_per_s": round(bps / 1e12, 3), "share_of_datasheet_hbm_bw": round(bps / DATASHEET_HBM_BPS, 3)}
    row["accumulate_over_store_time"] = round(row["accumulate"]["us_per_pass_median"] / row["store"]["us_per_pass_median"], 3)
    results["stage1"]["vgg16"] = row
    assert comm.status() == 0 and bool(torch.isfinite(partials).all())
    comm.close()


def end_to_end(args, results):
    from bagua_net_b200.models import build_model
    from bagua_net_b200.parallel import BnetDDP

    engines, data = {}, {}
    for k in args.ks:
        torch.manual_seed(0)
        model = build_model("vgg16", fused=True).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
        eng = BnetDDP(model, lr=0.01, momentum=0.9, weight_decay=1e-4, bucket_mb=64.0, accumulation_steps=k)
        eng.enable_cuda_graph(True)
        b = args.micro_batch * k
        x = torch.randn(b, 3, 224, 224, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 1000, (b,), device="cuda")
        for _ in range(args.warmup):
            eng.train_step(x, y)
        engines[k], data[k] = eng, (x, y)
    torch.cuda.synchronize()
    imgs = {k: [] for k in engines}
    for _ in range(args.e2e_rounds):
        for k, eng in engines.items():
            x, y = data[k]
            steps = max(2, args.e2e_images // x.shape[0])
            us = timed(lambda: eng.train_step(x, y), steps)
            imgs[k].append(x.shape[0] / (us * 1e-6))
    base = None
    for k, v in imgs.items():
        v = sorted(v)
        med = v[len(v) // 2]
        base = base or med
        results["end_to_end"][f"k{k}"] = {"global_batch": args.micro_batch * k, "img_per_s_median": round(med, 1),
                                          "img_per_s_min": round(v[0], 1), "img_per_s_max": round(v[-1], 1),
                                          "over_k1": round(med / base, 3)}
        assert engines[k].comm.status() == 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/grad_accum_step")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--micro-batch", type=int, default=32)
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--e2e-images", type=int, default=1024, help="images per timed window and variant")
    ap.add_argument("--e2e-rounds", type=int, default=5)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("grad_accum_step.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    results = {"card": card(), "bucket_mb": 64, "param_dtype": "bf16", "steps_per_window": args.steps, "rounds": args.rounds,
               "bytes_per_param": BYTES_PER_PARAM, "datasheet_hbm_tb_per_s": DATASHEET_HBM_BPS / 1e12, "stage1": {},
               "end_to_end": {}}
    stage1_times(args, results)
    if not args.no_e2e:
        end_to_end(args, results)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "grad_accum_step.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(results))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""What the EMA of the master weights costs in the fused data-parallel step, on one GPU.

1. The EMA launches of one optimizer step (one bnet_ema_update per bucket, then bnet_ema_advance) at the parameter counts
   of VGG16 (138.4 M) and ResNet-50 (25.6 M), bf16 parameters in 64 MB buckets, so one GPU's fp32 shards are whole
   buckets:
   * update: every step is an EMA step (ema_every=1), each launch lerps its shard;
   * skip: no step is an EMA step (ema_every=2^24), each launch reads the block and exits.
   Each path's step is captured in a CUDA graph, as the engine's captured step holds it, so the host's launch cost is not
   measured; CUDA events time `--steps` replays after `--warmup`, the two paths alternating for `--rounds` rounds
   (median).
   Bytes from the algorithm: 12 per shard element on the update path (master read, EMA read and written, fp32).  At the
   data sheet's 3.35 TB/s, VGG16 needs at least 0.50 ms per EMA step: a bound, not a measurement.
2. End to end: BnetDDP.train_step img/s on VGG16, bf16, batch `--batch`, 224 x 224, under a CUDA graph, with the EMA off,
   ema_every=1 and ema_every=32, alternating for `--e2e-rounds` rounds.

  python bench/ema_step.py --out profiles/ema_step
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))      # (`bench` is also bench.py at the root)
from optimizer_step import DATASHEET_HBM_BPS, MODELS, buckets, card  # noqa: E402
from bagua_net_b200.models import build_model  # noqa: E402
from bagua_net_b200.parallel import SymmComm  # noqa: E402

BYTES_PER_ELEMENT = 12
DECAY = 0.9998


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / steps


def ema_times(args, results):
    comm = SymmComm(64 << 20)
    for model, n in MODELS.items():
        sizes = buckets(n)
        master = [torch.randn(s, device="cuda") * 0.02 for s in sizes]
        ema = [m + torch.randn_like(m) * 1e-4 for m in master]
        # {1 - decay, every, step, n_averaged}: every step a lerp / no step an EMA step
        blocks = {"update": torch.tensor([1.0 - DECAY, 1.0, 0.0, 1.0], device="cuda"),
                  "skip": torch.tensor([1.0 - DECAY, float(1 << 24), 0.0, 1.0], device="cuda")}

        def step(blk):
            for m, e in zip(master, ema):
                comm.ema_update(m, e, blk)
            comm.ema_advance(blk)

        graphs = {}
        for k, blk in blocks.items():
            step(blk)                                     # (module load outside the capture)
            torch.cuda.synchronize()
            graphs[k] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphs[k]):
                step(blk)
            for _ in range(args.warmup):
                graphs[k].replay()
        torch.cuda.synchronize()
        times = {k: [] for k in blocks}
        for _ in range(args.rounds):
            for k, g in graphs.items():
                times[k].append(timed(g.replay, args.steps))
        elems = sum(sizes)
        row = {"params": n, "buckets": len(sizes), "shard_elements": elems,
               "update_bound_us_at_datasheet_bw": round(BYTES_PER_ELEMENT * elems / DATASHEET_HBM_BPS * 1e6, 1)}
        for k, ts in times.items():
            ts = sorted(ts)
            us = ts[len(ts) // 2]
            row[k] = {"us_per_step_median": round(us, 1), "us_per_step_min": round(ts[0], 1), "us_per_step_max": round(ts[-1], 1)}
            if k == "update":
                bps = BYTES_PER_ELEMENT * elems / (us * 1e-6)
                row[k].update(achieved_tb_per_s=round(bps / 1e12, 3), share_of_datasheet_hbm_bw=round(bps / DATASHEET_HBM_BPS, 3))
        # the counters ran on the device: every update-path step counted, no skip-path step averaged
        assert blocks["update"][3].item() == 1.0 + blocks["update"][2].item() and blocks["skip"][3].item() == 1.0
        assert bool(torch.isfinite(torch.cat(ema)).all())
        results["ema"][model] = row
        del master, ema
        torch.cuda.empty_cache()
    assert comm.status() == 0
    comm.close()


def end_to_end(args, results):
    from bagua_net_b200.parallel import BnetDDP

    x = torch.randn(args.batch, 3, 224, 224, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (args.batch,), device="cuda")
    engines = {}
    for name, kw in (("off", {}), ("every_1", {"ema_decay": DECAY, "ema_every": 1}),
                     ("every_32", {"ema_decay": DECAY, "ema_every": 32})):
        torch.manual_seed(1234)
        model = build_model("vgg16", fused=True).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
        eng = BnetDDP(model, lr=0.01, momentum=0.9, weight_decay=1e-4, bucket_mb=64.0, extra_heap_bytes=384 << 20, **kw)
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
    off = results["end_to_end"]["off"]["img_per_s_median"]
    for k in ("every_1", "every_32"):
        results["end_to_end"][f"{k}_over_off_img_per_s"] = round(results["end_to_end"][k]["img_per_s_median"] / off, 4)
    results["end_to_end"]["ema_n_averaged"] = {k: int(e._ema[3]) for k, e in engines.items() if e._ema is not None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/ema_step")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--e2e-steps", type=int, default=30)
    ap.add_argument("--e2e-rounds", type=int, default=5)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ema_step.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    results = {"card": card(), "bucket_mb": 64, "param_dtype": "bf16", "steps_per_window": args.steps, "rounds": args.rounds,
               "bytes_per_shard_element": BYTES_PER_ELEMENT, "datasheet_hbm_tb_per_s": DATASHEET_HBM_BPS / 1e12, "ema": {},
               "end_to_end": {}}
    ema_times(args, results)
    if not args.no_e2e:
        end_to_end(args, results)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "ema_step.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(results))


if __name__ == "__main__":
    main()

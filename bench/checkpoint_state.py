#!/usr/bin/env python
"""What saving and loading the layout-free optimizer state costs: BnetDDP.full_optimizer_state_dict() and
load_full_optimizer_state_dict() for VGG16's parameters (138.4 M) in bf16, AdamW with an EMA of the weights, 64 MB
buckets: 4 fp32 tensors per parameter (master, exp_avg, exp_avg_sq, EMA), 2.2 GB of state.

At one GPU and at the machine's GPU count (when above one), one process per GPU.  Each rank builds the engine (no
training: the times do not depend on the values), then `--rounds` times, behind a barrier:
* save: full_optimizer_state_dict() on every rank (rank 0 receives the dict in host memory), wall clock to the last rank;
* load: every rank calls load_full_optimizer_state_dict() with a copy of that dict loaded from a file (torch.load with
  map_location="cpu", not timed), wall clock to the last rank.
The median, min and max over rounds are printed as one JSON line with the card's name and power limit.

  python bench/checkpoint_state.py [--rounds 3] [--out DIR]
"""
import argparse
import json
import os
import shutil
import socket
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))      # (`bench` is also bench.py at the root)


def worker(args):
    import torch.distributed as dist

    from bagua_net_b200.models import build_model
    from bagua_net_b200.parallel import BnetDDP, init_process_group_from_env

    init_process_group_from_env()
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    model = build_model("vgg16", fused=True).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    eng = BnetDDP(model, optimizer="adamw", lr=1e-3, weight_decay=0.05, ema_decay=0.9999, bucket_mb=64.0)

    def sync():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()

    path = os.path.join(args.tmp, "state.pt")
    save, load = [], []
    for _ in range(args.rounds):
        sync()
        t0 = time.perf_counter()
        full = eng.full_optimizer_state_dict()
        sync()
        save.append(time.perf_counter() - t0)
        if rank == 0:
            torch.save(full, path)
        del full
        sync()
        state = torch.load(path, map_location="cpu")
        sync()
        t0 = time.perf_counter()
        eng.load_full_optimizer_state_dict(state)
        sync()
        load.append(time.perf_counter() - t0)
        del state
    if rank == 0:
        from optimizer_step import card

        nbytes = 4 * 4 * sum(p.numel() for p in eng._params)
        row = {"world": world, "buckets": len(eng.buckets), "params": sum(p.numel() for p in eng._params),
               "state_bytes": nbytes, "card": card()}
        for k, ts in (("save", save), ("load", load)):
            ts = sorted(ts)
            row[k] = {"s_median": round(ts[len(ts) // 2], 3), "s_min": round(ts[0], 3), "s_max": round(ts[-1], 3),
                      "gb_per_s_median": round(nbytes / ts[len(ts) // 2] / 1e9, 2)}
        print("RESULT " + json.dumps(row), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def run(world, args):
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    procs = []
    for r in range(world):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
        procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), "--worker", "--rounds", str(args.rounds),
                                       "--tmp", args.tmp], env=env, stdout=subprocess.PIPE, text=True))
    outs = [p.communicate(timeout=1800)[0] for p in procs]
    if any(p.returncode for p in procs):
        raise SystemExit(f"world {world}: a rank failed\n{outs[0][-4000:]}")
    return json.loads([ln for ln in outs[0].splitlines() if ln.startswith("RESULT ")][-1][7:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="", help="also write checkpoint_state.json into this directory")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--tmp", default="", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    if not torch.cuda.is_available():
        raise SystemExit("checkpoint_state.py measures on a GPU; none is visible")
    n = torch.cuda.device_count()
    results = {"model": "vgg16", "param_dtype": "bf16", "optimizer": "adamw+ema", "bucket_mb": 64, "rounds": args.rounds,
               "runs": []}
    args.tmp = tempfile.mkdtemp(prefix="bnet-ckpt-bench-")
    try:
        for world in sorted({1, n}):
            results["runs"].append(run(world, args))
    finally:
        shutil.rmtree(args.tmp, ignore_errors=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "checkpoint_state.json"), "w") as f:
            json.dump(results, f, indent=1)
    print(json.dumps(results))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""All-reduce bus-bandwidth sweep 1 KB – 1 GB (BASELINE.json config #5): the fused bnet kernels
(NVLS multimem / NVLink P2P / one-shot) against stock NCCL on the same box, device-timed with CUDA
events, max over ranks, reported against the NVLink roofline.

  python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
      bench/allreduce_sweep.py [--min-bytes 1K --max-bytes 1G --dtype bf16 --blocks 0 --json out.json]

Roofline: an in-switch (NVLS) all-reduce of S bytes moves S(1+1/n) bytes in and out of every GPU;
a P2P two-shot moves 2S(n-1)/n.  Link bandwidth = 450 GB/s per direction per GPU, the nominal NVLink 4 figure of an
H100 SXM (data sheet; not a measured peak).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bagua_net_b200.parallel import SymmComm, init_process_group_from_env  # noqa: E402

LINK_GBS = 450.0          # nominal, H100 SXM NVLink 4 per direction


def parse_size(s: str) -> int:
    s = s.strip().upper()
    mult = {"K": 1 << 10, "M": 1 << 20, "G": 1 << 30}.get(s[-1], 1)
    return int(float(s[:-1]) * mult) if s[-1] in "KMG" else int(s)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-bytes", default="1K")
    ap.add_argument("--max-bytes", default="1G")
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "f32", "f16"])
    ap.add_argument("--blocks", default="0", help="comma list of CTA counts to try for the bnet kernels (0 = default)")
    ap.add_argument("--algos", default="nvls,p2p,oneshot,nccl")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default="")
    a = ap.parse_args()

    init_process_group_from_env("nccl")
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = torch.device("cuda", torch.cuda.current_device())
    dtype = {"bf16": torch.bfloat16, "f32": torch.float32, "f16": torch.float16}[a.dtype]
    es = torch.empty((), dtype=dtype).element_size()
    lo, hi = parse_size(a.min_bytes), parse_size(a.max_bytes)
    comm = SymmComm(hi + (64 << 20))
    algos = [x for x in a.algos.split(",") if x]
    if not comm.has_multicast and "nvls" in algos:
        algos.remove("nvls")
    blocks = [int(b) for b in a.blocks.split(",")]
    buf = comm.alloc(hi // es, dtype)
    plain = torch.empty(hi // es, dtype=dtype, device=dev)
    out1 = torch.empty(min(hi, 8 << 20) // es, dtype=dtype, device=dev)
    buf.fill_(1)
    plain.fill_(1)

    def timed(fn, iters):
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1) / iters], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item()) * 1e3   # us

    rows = []
    if rank == 0:
        print(f"# world {world} dtype {a.dtype} multicast {comm.has_multicast}  (us, algbw GB/s, busbw GB/s, fraction of {LINK_GBS:.0f} GB/s roofline)")
        print(f"#{'bytes':>12s} {'algo':>10s} {'ctas':>5s} {'time_us':>10s} {'algbw':>8s} {'busbw':>8s} {'roofline':>8s}")
    quantum = 16 * world
    size = lo
    while size <= hi:
        nbytes = max(quantum, size // quantum * quantum)
        n = nbytes // es
        iters = a.iters if nbytes <= (64 << 20) else max(5, a.iters // 4)
        for algo in algos:
            for nb in (blocks if algo != "nccl" else [0]):
                if algo == "oneshot" and nbytes > (8 << 20):
                    continue
                if algo == "nccl":
                    us = timed(lambda: dist.all_reduce(plain[:n]), iters)
                elif algo == "oneshot":
                    us = timed(lambda: comm.all_reduce_oneshot(buf[:n], out1[:n], "sum", nblocks=nb), iters)
                else:
                    us = timed(lambda: comm.all_reduce(buf[:n], "sum", algo=algo, nblocks=nb), iters)
                algbw = nbytes / us / 1e3
                busbw = algbw * 2 * (world - 1) / world
                # time lower bound per algorithm at link bandwidth
                # bytes per direction per GPU: NVLS S(1+1/n); direct two-shot S(n-1)/n (peer loads in,
                # peer stores out, full duplex); one-shot S(n-1) in; NCCL ring 2S(n-1)/n
                moved = {"nvls": nbytes * (1 + 1 / world), "p2p": nbytes * (world - 1) / world,
                         "oneshot": nbytes * (world - 1)}.get(algo, nbytes * 2 * (world - 1) / world)
                frac = (moved / (LINK_GBS * 1e3)) / us
                rows.append({"bytes": nbytes, "algo": algo, "ctas": nb, "us": us, "algbw": algbw, "busbw": busbw, "roofline_frac": frac})
                if rank == 0:
                    print(f"{nbytes:>13d} {algo:>10s} {nb:>5d} {us:>10.1f} {algbw:>8.1f} {busbw:>8.1f} {frac:>8.3f}", flush=True)
        size *= 2 if size < (1 << 20) else 4 if size < (64 << 20) else 2
    if rank == 0 and a.json:
        with open(a.json, "w") as f:
            json.dump({"world": world, "dtype": a.dtype, "multicast": comm.has_multicast, "link_gbs": LINK_GBS, "rows": rows}, f)
    assert comm.status() == 0
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

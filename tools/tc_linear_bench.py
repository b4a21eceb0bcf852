"""wgmma linear (csrc/cuda/tc_gemm.cu) against cuBLAS at the flagship's classifier shapes and a few square ones:
CUDA-event timed, TFLOP/s against the H100 SXM's data-sheet dense bf16 rate, GB/s for the weight-streaming small-batch
shapes.

    python tools/tc_linear_bench.py [--shapes MxNxK,...] [--iters 20]
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bagua_net_b200.ops import tc_linear  # noqa: E402

DEFAULT = "32x4096x25088,32x4096x4096,32x1000x4096,256x4096x4096,1024x4096x4096,4096x4096x4096,8192x8192x8192"


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3   # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default=DEFAULT)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    peak_tf, peak_bw = 989.0, 3350.0      # H100 SXM dense bf16 TFLOP/s and HBM3 GB/s, data sheet (700 W), not measured peaks
    if not tc_linear.supported():
        print("wgmma linear unsupported here")
        return 1
    print(f"# cuBLAS bf16 peak {peak_tf:.0f} TFLOP/s, HBM copy rate {peak_bw:.0f} GB/s")
    print(f"# {'M x N x K':>22s} {'ours us':>9s} {'TF/s':>7s} {'GB/s':>7s} {'cuBLAS us':>10s} {'TF/s':>7s} {'ours/cuBLAS':>11s} {'max err':>8s}")
    for shp in a.shapes.split(","):
        M, N, K = (int(v) for v in shp.split("x"))
        x = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        y = tc_linear.linear(x, w, b, True)
        flag = tc_linear.last_error()
        ref = torch.relu(torch.nn.functional.linear(x, w, b))
        err = (y.float() - ref.float()).abs().max().item()
        t_ours = timed(lambda: tc_linear.linear(x, w, b, True, out=y), a.iters, a.warmup)
        t_one = timed(lambda: tc_linear.linear(x, w, b, True, out=y, splits=1), a.iters, a.warmup) if M <= 64 else t_ours
        t_ref = timed(lambda: torch.relu_(torch.nn.functional.linear(x, w, b)), a.iters, a.warmup)
        flops = 2.0 * M * N * K
        nbytes = 2.0 * (M * K + N * K + M * N)
        print(f"  {shp:>22s} {t_ours:9.1f} {flops / t_ours / 1e6:7.0f} {nbytes / t_ours / 1e3:7.0f} {t_ref:10.1f} "
              f"{flops / t_ref / 1e6:7.0f} {t_ref / t_ours:11.2f} {err:8.4f}" + (f"  (no split-K: {t_one:.1f} us)" if M <= 64 else "")
              + (f"  WATCHDOG {flag}" if flag else ""))
    return 0


if __name__ == "__main__":
    sys.exit(main())

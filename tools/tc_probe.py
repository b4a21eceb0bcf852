"""First-contact diagnostics for the wgmma linear kernel (csrc/cuda/tc_gemm.cu): structured inputs whose products say
WHICH part of the data path is wrong when the numerics test fails — instead of "max abs err 3.7".

    python tools/tc_probe.py            # prints one verdict per probe; exit code 1 if any failed

Probes (all exact in bf16 / fp32, so any mismatch is a layout or synchronisation bug, not rounding):
  rows      D[i, j] = i          -> accumulator row <-> output row mapping of the consumer warps
  cols      D[i, j] = j          -> accumulator column <-> output column mapping, wgmma register order
  kslice    only k in [16s, 16s+16) non-zero, for every s in a 64-wide K block
                                 -> the +32-byte descriptor advance inside the 128-byte swizzle row
  kblock    only K block b non-zero -> ring stage / phase bookkeeping, TMA coordinates
  swz       A[i, k] = 1 iff k == (i * 7) % 64  (a different column per row), B[j, k] = k
                                 -> TMA swizzle vs. UMMA descriptor swizzle agree (D[i, j] = (i * 7) % 64)
  ragged    M, N, K off the tile grid -> TMA zero fill and the epilogue guards
  dgrad / wgrad  the MN-major operand path (64 x 64 boxes, LBO / SBO of the MN-major descriptor), exact integers
  tiles     many tiles per CTA (persistent loop, both accumulator stages), checked tile by tile
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bagua_net_b200.ops import tc_linear  # noqa: E402

FAILED = []


def run(name, x, w, expect=None, detail=None):
    y = tc_linear.linear(x.bfloat16().contiguous(), w.bfloat16().contiguous()).float()
    flag = tc_linear.last_error()
    ref = (x.double() @ w.double().t()).float() if expect is None else expect
    ref = ref.bfloat16().float()                 # the kernel rounds its fp32 accumulator to bf16 (nearest even), like torch
    bad = (y != ref)
    ok = flag == 0 and not bool(bad.any())
    msg = f"[{'ok' if ok else 'FAIL'}] {name}: M={x.shape[0]} N={w.shape[0]} K={x.shape[1]}"
    if flag:
        msg += f"  watchdog role {flag} (1 = TMA producer, 2 = MMA issuer, 3 = epilogue)"
    if bool(bad.any()):
        idx = bad.nonzero()
        rows, cols = idx[:, 0].unique(), idx[:, 1].unique()
        msg += (f"  {int(bad.sum())} wrong of {bad.numel()}; rows {rows[:8].tolist()}{'...' if len(rows) > 8 else ''}"
                f" cols {cols[:8].tolist()}{'...' if len(cols) > 8 else ''}")
        i, j = idx[0].tolist()
        msg += f"; first: D[{i},{j}] = {y[i, j].item()} expected {ref[i, j].item()}"
        if detail:
            msg += "  " + detail(y, ref)
    print(msg)
    if not ok:
        FAILED.append(name)
    return y


def main():
    if not tc_linear.supported():
        print("wgmma linear unsupported on this device / driver")
        return 1
    dev = "cuda"
    for (M, N) in ((128, 128), (32, 128)):                  # plain and swapped orientation, one tile each
        tag = "swap" if M <= 64 else "noswap"
        K = 64
        k0 = 5
        # rows: x[i, k0] = i, w[j, k0] = 1
        x = torch.zeros(M, K, device=dev); w = torch.zeros(N, K, device=dev)
        x[:, k0] = torch.arange(M, device=dev).float(); w[:, k0] = 1
        run(f"rows/{tag}", x, w)
        # cols: x[i, k0] = 1, w[j, k0] = j
        x = torch.zeros(M, K, device=dev); w = torch.zeros(N, K, device=dev)
        x[:, k0] = 1; w[:, k0] = torch.arange(N, device=dev).float()
        run(f"cols/{tag}", x, w)
        # kslice: which 16-wide slice of the K block reaches the MMA
        for s in range(4):
            x = torch.zeros(M, K, device=dev); w = torch.zeros(N, K, device=dev)
            x[:, 16 * s:16 * s + 16] = 1; w[:, 16 * s:16 * s + 16] = 1
            run(f"kslice{s}/{tag}", x, w)                    # expect 16 everywhere
        # swizzle agreement: a different k per row
        x = torch.zeros(M, K, device=dev)
        x[torch.arange(M), (torch.arange(M) * 7) % 64] = 1
        w = torch.arange(K, device=dev).float().repeat(N, 1)
        run(f"swz/{tag}", x, w)
        # kblock: 8 K blocks, only block b carries data (value b + 1)
        K = 512
        for b in (0, 1, 5, 6, 7):
            x = torch.zeros(M, K, device=dev); w = torch.zeros(N, K, device=dev)
            x[:, 64 * b] = b + 1; w[:, 64 * b] = 1
            run(f"kblock{b}/{tag}", x, w)
        # everything at once, exact small integers
        g = torch.Generator(device=dev).manual_seed(1)
        x = torch.randint(-2, 3, (M, K), device=dev, generator=g).float()
        w = torch.randint(-2, 3, (N, K), device=dev, generator=g).float()
        run(f"ints/{tag}", x, w)
    # ragged shapes
    g = torch.Generator(device=dev).manual_seed(2)
    for (M, N, K) in ((130, 136, 72), (48, 200, 264), (1, 8, 8), (257, 129, 1000)):
        x = torch.randint(-2, 3, (M, K), device=dev, generator=g).float()
        w = torch.randint(-2, 3, (N, K), device=dev, generator=g).float()
        run("ragged", x, w)
    # backward GEMMs (MN-major operands): exact integers, both orientations of dX
    for (M, N, K) in ((128, 128, 128), (32, 128, 128), (256, 192, 320), (48, 200, 264)):
        gy = torch.randint(-2, 3, (M, N), device=dev, generator=g).float()
        w = torch.randint(-2, 3, (N, K), device=dev, generator=g).float()
        x = torch.randint(-2, 3, (M, K), device=dev, generator=g).float()
        for name, got, ref in (("dgrad", tc_linear.linear_dgrad(gy.bfloat16(), w.bfloat16()), gy @ w),
                               ("wgrad", tc_linear.linear_wgrad(gy.bfloat16(), x.bfloat16()), gy.t() @ x)):
            flag = tc_linear.last_error()
            bad = got.float() != ref.bfloat16().float()
            ok = flag == 0 and not bool(bad.any())
            msg = f"[{'ok' if ok else 'FAIL'}] {name}: M={M} N={N} K={K}"
            if flag:
                msg += f"  watchdog role {flag}"
            if bool(bad.any()):
                idx = bad.nonzero()
                msg += (f"  {int(bad.sum())} wrong of {bad.numel()}; rows {idx[:, 0].unique()[:8].tolist()} cols "
                        f"{idx[:, 1].unique()[:8].tolist()}; first D{idx[0].tolist()} = "
                        f"{got[idx[0][0], idx[0][1]].item()} expected {ref[idx[0][0], idx[0][1]].item()}")
            print(msg)
            if not ok:
                FAILED.append(name)
    # persistent loop: far more tiles than SMs; report the first wrong TILE
    M, N, K = 4096, 8192, 192
    x = torch.randint(-2, 3, (M, K), device=dev, generator=g).float()
    w = torch.randint(-2, 3, (N, K), device=dev, generator=g).float()
    p = tc_linear.plan(M, N, K)

    def tiles(y, ref):
        bad = (y != ref).view(M // 128, 128, N // p["bn"], p["bn"]).any(3).any(1)
        t = bad.nonzero()
        return f"{int(bad.sum())} of {bad.numel()} tiles wrong; first (row block, col block) = {t[0].tolist()}; plan {p}"

    run("tiles", x, w, detail=tiles)
    print("FAILED: " + ", ".join(FAILED) if FAILED else "all probes passed")
    return 1 if FAILED else 0


if __name__ == "__main__":
    sys.exit(main())

"""Stand-alone bandwidth check of the fused layer kernels (csrc/cuda/nn_kernels.cu) at the VGG16 shapes of the
flagship benchmark (batch 32, bf16, NHWC): every kernel alone on the GPU, CUDA-event timed, bytes counted from the
tensors it reads and writes, reported against the H100 SXM's nominal HBM3 bandwidth (3.35 TB/s, data sheet).

    python tools/nn_kernel_bench.py [--batch 32] [--iters 20]
    ncu --set full --clock-control none --import-source on -k "regex:relu_bwd|pool_relu_bwd|bias_relu" \
        -o gpurun_out/nn_kernels python tools/nn_kernel_bench.py --iters 1 --warmup 0
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bagua_net_b200.ops import fused_nn  # noqa: E402

# (C_out, H=W of the conv output, pooled?) for the 13 conv layers of VGG16 at 224x224
VGG16 = [(64, 224, False), (64, 224, True), (128, 112, False), (128, 112, True), (256, 56, False), (256, 56, False),
         (256, 56, True), (512, 28, False), (512, 28, False), (512, 28, True), (512, 14, False), (512, 14, False),
         (512, 14, True)]


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
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    peak = 3350.0          # H100 SXM HBM3, data sheet (not a measured copy rate)
    L = fused_nn._L()
    st = fused_nn._stream
    dt = torch.bfloat16
    N = a.batch
    tot = {}
    print(f"# batch {N} bf16 NHWC; nominal HBM3 {peak:.0f} GB/s; per kernel: us, GB/s, fraction of it")
    print(f"# {'kernel':28s} {'C':>4s} {'HxW':>8s} {'MB':>8s} {'us':>8s} {'GB/s':>8s} {'frac':>6s}")
    for c, hw, pool in VGG16:
        rows = N * hw * hw
        z = torch.randn(N, c, hw, hw, device="cuda", dtype=dt).contiguous(memory_format=torch.channels_last)
        b = torch.randn(c, device="cuda", dtype=dt)
        gb = torch.zeros(c, device="cuda", dtype=torch.float32)
        part1 = fused_nn._partials(c, gb.device)
        nbytes = rows * c * 2
        if not pool:
            y = torch.relu(z)
            gy = torch.randn_like(z)
            gz = torch.empty_like(z)
            cases = [
                ("bias_relu (fwd)", 2 * nbytes, lambda: L.bnet_nn_bias_relu(z.data_ptr(), b.data_ptr(), rows, c, 1, st())),
                ("relu_bwd_bias_grad", 3 * nbytes,
                 lambda: L.bnet_nn_relu_bwd_bias_grad(gy.data_ptr(), y.data_ptr(), gz.data_ptr(), gb.data_ptr(), part1.data_ptr(), rows, c, 1, st())),
            ]
        else:
            p = torch.empty((N, c, hw // 2, hw // 2), device="cuda", dtype=dt, memory_format=torch.channels_last)
            idx = torch.empty(rows // 4 * c, device="cuda", dtype=torch.uint8)
            gp = torch.randn_like(p)
            gz = torch.empty_like(z)
            L.bnet_nn_bias_relu_pool_fwd(z.data_ptr(), b.data_ptr(), p.data_ptr(), idx.data_ptr(), N, hw, hw, c, 1, st())
            cases = [
                ("bias_relu_pool_fwd", nbytes + nbytes // 4 + nbytes // 8,
                 lambda: L.bnet_nn_bias_relu_pool_fwd(z.data_ptr(), b.data_ptr(), p.data_ptr(), idx.data_ptr(), N, hw, hw, c, 1, st())),
                ("pool_relu_bwd_bias_grad", nbytes + nbytes // 4 + nbytes // 8,
                 lambda: L.bnet_nn_pool_relu_bwd_bias_grad(gp.data_ptr(), idx.data_ptr(), gz.data_ptr(), gb.data_ptr(), part1.data_ptr(), N, hw, hw, c, 1, st())),
            ]
        for name, traffic, fn in cases:
            us = timed(fn, a.iters, a.warmup)
            gbs = traffic / us / 1e3
            t = tot.setdefault(name, [0.0, 0.0])
            t[0] += traffic
            t[1] += us
            print(f"  {name:28s} {c:4d} {hw:4d}x{hw:<3d} {traffic / 1e6:8.1f} {us:8.1f} {gbs:8.0f} {gbs / peak:6.2f}")
        del z
    # ---- BatchNorm family at the ResNet-50 shapes (C, H=W of the convolution output)
    RESNET = [(64, 112), (64, 56), (256, 56), (128, 28), (512, 28), (256, 14), (1024, 14), (512, 7), (2048, 7)]
    vp, ll, i, f = fused_nn.C.c_void_p, fused_nn.C.c_longlong, fused_nn.C.c_int, fused_nn.C.c_float
    print("# BatchNorm family (stats, apply+ReLU+residual, backward reduce, backward apply)")
    for c, hw in RESNET:
        rows = N * hw * hw
        z = torch.randn(N, c, hw, hw, device="cuda", dtype=dt).contiguous(memory_format=torch.channels_last)
        res, gy = torch.randn_like(z), torch.randn_like(z)
        y, gz, gres = torch.empty_like(z), torch.empty_like(z), torch.empty_like(z)
        gamma, beta = torch.ones(c, device="cuda", dtype=dt), torch.zeros(c, device="cuda", dtype=dt)
        rm, rv = torch.zeros(c, device="cuda", dtype=dt), torch.ones(c, device="cuda", dtype=dt)
        dg, db = torch.empty_like(gamma), torch.empty_like(gamma)
        stats = torch.zeros(2 * c, device="cuda", dtype=torch.float32)
        gsum = torch.zeros(2 * c, device="cuda", dtype=torch.float32)
        part2 = fused_nn._partials(2 * c, gsum.device)
        nbytes = rows * c * 2
        L.bnet_nn_bn_stats(z.data_ptr(), stats.data_ptr(), part2.data_ptr(), rows, c, 1, st())
        cases = [
            ("bn_stats", nbytes, lambda: L.bnet_nn_bn_stats(z.data_ptr(), stats.data_ptr(), part2.data_ptr(), rows, c, 1, st())),
            ("bn_apply(+res+relu)", 3 * nbytes, lambda: L.bnet_nn_bn_apply(z.data_ptr(), res.data_ptr(), y.data_ptr(), stats.data_ptr(),
                                                                          gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr(),
                                                                          rows, c, 1e-5, 0.1, 1, 1, st())),
            ("bn_bwd_reduce", 3 * nbytes, lambda: L.bnet_nn_bn_bwd_reduce(gy.data_ptr(), y.data_ptr(), z.data_ptr(), stats.data_ptr(),
                                                                         gsum.data_ptr(), part2.data_ptr(), rows, c, 1e-5, 1, 1, st())),
            ("bn_bwd_apply(+gres)", 5 * nbytes, lambda: L.bnet_nn_bn_bwd_apply(gy.data_ptr(), y.data_ptr(), z.data_ptr(), gz.data_ptr(),
                                                                              gres.data_ptr(), stats.data_ptr(), gsum.data_ptr(),
                                                                              gamma.data_ptr(), dg.data_ptr(), db.data_ptr(), rows, c,
                                                                              1e-5, 1, 1, st())),
        ]
        for name, traffic, fn in cases:
            us = timed(fn, a.iters, a.warmup)
            gbs = traffic / us / 1e3
            t = tot.setdefault(name, [0.0, 0.0])
            t[0] += traffic
            t[1] += us
            print(f"  {name:28s} {c:4d} {hw:4d}x{hw:<3d} {traffic / 1e6:8.1f} {us:8.1f} {gbs:8.0f} {gbs / peak:6.2f}")
    print("# totals over the listed layers:")
    for name, (traffic, us) in tot.items():
        print(f"  {name:28s} {traffic / 1e6:9.1f} MB {us:9.1f} us {traffic / us / 1e3:8.0f} GB/s {traffic / us / 1e3 / peak:6.2f}")


if __name__ == "__main__":
    main()

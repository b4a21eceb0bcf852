"""wgmma 3x3 convolution (csrc/cuda/tc_gemm.cu, kConv) against cuDNN at the flagship's layer shapes: forward with
bias + ReLU (ours: one kernel; library: cuDNN convolution + our in-place bias/ReLU pass), the input gradient and the
filter gradient (--wgrad; ours: 64-pixel 4-D TMA boxes of gy and x, split over the pixels).
CUDA-event timed; TFLOP/s against the H100 SXM's data-sheet dense bf16 rate (989 TFLOP/s at 700 W).

    python tools/tc_conv_bench.py [--batch 32] [--iters 10] [--model vgg16|resnet]
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bagua_net_b200.ops import fused_nn, tc_conv, tc_linear  # noqa: E402

VGG = [(64, 64, 224), (64, 128, 112), (128, 128, 112), (128, 256, 56), (256, 256, 56), (256, 512, 28), (512, 512, 28), (512, 512, 14)]
RESNET = [(64, 64, 56), (128, 128, 28), (256, 256, 14), (512, 512, 7)]


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--model", default="vgg16")
    ap.add_argument("--shapes", default="")
    ap.add_argument("--wgrad", action="store_true", help="also time the filter gradient (ours vs cuDNN), with the splits ours used")
    args = ap.parse_args()
    peak = 989.0           # H100 SXM dense bf16, data sheet (700 W)
    shapes = VGG if args.model.startswith("vgg") else RESNET
    if args.shapes:
        shapes = [tuple(int(v) for v in s.split("x")) for s in args.shapes.split(",")]
    assert tc_linear.supported()
    print(f"# batch {args.batch}, bf16 NHWC, 3x3 s1 p1; cuBLAS bf16 sustained {peak:.0f} TFLOP/s")
    print(f"#{'cin':>5} {'cout':>5} {'hw':>4} | {'fwd ours':>9} {'TF/s':>6} {'cudnn+br':>9} {'TF/s':>6} {'ratio':>6} | "
          f"{'dgrad ours':>10} {'TF/s':>6} {'cudnn':>8} {'TF/s':>6} {'ratio':>6} | max err")
    n = args.batch
    for cin, cout, hw in shapes:
        g = torch.Generator(device="cuda").manual_seed(1)
        x = torch.randn(n, cin, hw, hw, device="cuda", generator=g).bfloat16().contiguous(memory_format=torch.channels_last)
        w = (torch.randn(cout, cin, 3, 3, device="cuda", generator=g) / (3 * cin ** 0.5)).bfloat16().contiguous(memory_format=torch.channels_last)
        b = torch.randn(cout, device="cuda", generator=g).bfloat16()
        gy = torch.randn(n, cout, hw, hw, device="cuda", generator=g).bfloat16().contiguous(memory_format=torch.channels_last)
        flops = 2.0 * n * hw * hw * cin * cout * 9

        def lib_fwd():
            z = fused_nn._conv(x, w, [1, 1], [1, 1])
            fused_nn._chk(fused_nn._L().bnet_nn_bias_relu(z.data_ptr(), b.data_ptr(), n * hw * hw, cout, 1, fused_nn._stream()), "bias_relu")
            return z

        def lib_dgrad():
            return torch.ops.aten.convolution_backward(gy, x, w, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [True, False, False])[0]

        y_tc, y_lib = tc_conv.conv3x3(x, w, b, relu=True), lib_fwd()
        err = ((y_tc.float() - y_lib.float()).norm() / y_lib.float().norm()).item()
        t_tc = timed(lambda: tc_conv.conv3x3(x, w, b, relu=True), args.iters)
        t_lib = timed(lib_fwd, args.iters)
        if cout % 64 == 0:
            d_tc, d_lib = tc_conv.conv3x3_dgrad(gy, w), lib_dgrad()
            err = max(err, ((d_tc.float() - d_lib.float()).norm() / d_lib.float().norm()).item())
            t_dtc = timed(lambda: tc_conv.conv3x3_dgrad(gy, w), args.iters)
            t_dlib = timed(lib_dgrad, args.iters)
        else:
            t_dtc = t_dlib = float("nan")
        tf = lambda us: flops / us / 1e6      # noqa: E731
        extra = ""
        if args.wgrad and cin % 64 == 0 and cout % 64 == 0:
            def lib_wgrad():
                return torch.ops.aten.convolution_backward(gy, x, w, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [False, True, False])[1]

            w_tc, w_lib = tc_conv.conv3x3_wgrad(gy, x), lib_wgrad()
            werr = ((w_tc.float() - w_lib.float()).norm() / w_lib.float().norm()).item()
            t_wtc = timed(lambda: tc_conv.conv3x3_wgrad(gy, x), args.iters)
            t_wlib = timed(lib_wgrad, args.iters)
            p = tc_conv.wgrad_plan(n, hw, hw, cin, cout)
            extra = (f" | wgrad ours {t_wtc:7.1f} us {tf(t_wtc):5.0f} TF/s, cuDNN {t_wlib:7.1f} us {tf(t_wlib):5.0f} TF/s, ratio {t_wlib / t_wtc:5.2f}, "
                     f"err {werr:.4f} ({p['grid_x'] * p['grid_y']} tiles of 128x{p['bn']} x {p['grid_z']} pixel slices)")
        print(f" {cin:5d} {cout:5d} {hw:4d} | {t_tc:9.1f} {tf(t_tc):6.0f} {t_lib:9.1f} {tf(t_lib):6.0f} {t_lib / t_tc:6.2f} | "
              f"{t_dtc:10.1f} {tf(t_dtc):6.0f} {t_dlib:8.1f} {tf(t_dlib):6.0f} {t_dlib / t_dtc:6.2f} | {err:.4f}{extra}")
    print(f"# watchdog flag {tc_linear.last_error()}")


if __name__ == "__main__":
    main()

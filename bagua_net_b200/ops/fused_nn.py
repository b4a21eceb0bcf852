"""Fused conv-block layers (csrc/cuda/nn_kernels.cu): everything memory-bound that follows a
convolution is folded into one sm_90a pass in forward and one in backward.

    ConvBiasReLU      y = relu(conv(x, w) + b)
    ConvBiasReLUPool  p = maxpool2x2(relu(conv(x, w) + b))      (y is never written to HBM)

The convolution itself stays a library call (cuDNN implicit GEMM on the tensor cores); the bias
add, ReLU, 2x2 max-pool, their backward passes and the bias-gradient reduction are ours.
Inputs must be channels_last with C_out a multiple of 8 (bf16) / 4 (fp32); otherwise the layer
falls back to the eager PyTorch ops.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from ..utils.native import load

_DT = {torch.float32: 0, torch.bfloat16: 1}
LAUNCHES = 0          # kernels of ours launched by this module (bench.py reports it)
_lib = None


def _L():
    global _lib
    if _lib is None:
        _lib = load()
        vp, ll, i = C.c_void_p, C.c_longlong, C.c_int
        _lib.bnet_nn_bias_relu.argtypes = [vp, vp, ll, i, i, vp]
        _lib.bnet_nn_relu_bwd_bias_grad.argtypes = [vp, vp, vp, vp, vp, ll, i, i, vp]
        _lib.bnet_nn_bias_relu_pool_fwd.argtypes = [vp, vp, vp, vp, i, i, i, i, i, vp]
        _lib.bnet_nn_pool_relu_bwd_bias_grad.argtypes = [vp, vp, vp, vp, vp, i, i, i, i, i, vp]
        f = C.c_float
        _lib.bnet_nn_bn_stats.argtypes = [vp, vp, vp, ll, i, i, vp]
        _lib.bnet_nn_bn_apply.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, ll, i, f, f, i, i, vp]
        _lib.bnet_nn_bn_bwd_reduce.argtypes = [vp, vp, vp, vp, vp, vp, ll, i, f, i, i, vp]
        _lib.bnet_nn_bn_bwd_apply.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, ll, i, f, i, i, vp]
    return _lib


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _partials(ld: int, device) -> torch.Tensor:
    """Workspace of a column reduction: one row of `ld` block partial sums per block, added up in block order by the library
    (the same sums on every run); allocated on the current stream, so concurrent streams and graph captures get their own."""
    return torch.empty((_L().bnet_nn_partial_rows(), ld), device=device, dtype=torch.float32)


def _chk(rc, what):
    global LAUNCHES
    if rc < 0:
        raise RuntimeError(f"bnet kernel {what} failed (rc={rc})")
    LAUNCHES += rc


def _nhwc(t: torch.Tensor) -> bool:
    return t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last)


def _supported(x: torch.Tensor, cout: int) -> bool:
    return x.is_cuda and x.dtype in _DT and cout % (8 if x.dtype == torch.bfloat16 else 4) == 0


def _conv(x, w, stride, padding):
    return torch.ops.aten.convolution(x, w, None, stride, padding, [1, 1], False, [0, 0], 1)


def _conv_backward(gz, x, w, stride, padding, need_x):
    """(gx, gw) of the convolution.  For 3x3 / stride 1 / pad 1 layers the autotuner (ops/tc_conv.py) decides per shape and
    per gradient: the input gradient from the wgmma kernel (the filter is read as stored, MN-major, taps flipped), the
    filter gradient from the wgmma kernel (64-pixel boxes of gz and x, split over the pixels) — or cuDNN for either."""
    def lib(want_x, want_w):
        return torch.ops.aten.convolution_backward(gz, x, w, None, stride, padding, [1, 1], False, [0, 0], 1, [want_x, want_w, False])

    if _is_3x3_s1p1(w, stride, padding) and gz.dtype == torch.bfloat16:
        from . import tc_conv

        tc_x = need_x and tc_conv.choose("dgrad", gz, w, lambda: lib(True, False)[0], lambda: tc_conv.conv3x3_dgrad(gz, w),
                                         tc_conv.close) == "tc"
        tc_w = tc_conv.choose_wgrad(gz, x, w, lambda: lib(False, True)[1]) == "tc"
        if tc_x or tc_w:
            gx = tc_conv.conv3x3_dgrad(gz, w) if tc_x else None
            gw = None
            if tc_w:
                # the kernel writes the filter gradient straight into the parameter's slice of the engine's flat gradient
                # buffer when there is one (ops/grad_target.py); autograd adopts the slice instead of accumulating into it
                from . import grad_target

                dst = grad_target.lookup(w)
                gw = tc_conv.conv3x3_wgrad(gz, x, out=dst)
                if dst is not None and gw.data_ptr() == dst.data_ptr():
                    gw = grad_target.adopt(dst)
            if (need_x and gx is None) or gw is None:
                rx, rw, _ = lib(need_x and gx is None, gw is None)
                gx = rx if gx is None else gx
                gw = rw if gw is None else gw
            return gx, gw
    gx, gw, _ = lib(need_x, True)
    return gx, gw


_zeros: dict = {}


def _zero_bias(b: torch.Tensor) -> torch.Tensor:
    key = (b.device, b.dtype, b.numel())
    if key not in _zeros:
        _zeros[key] = torch.zeros_like(b)
    return _zeros[key]


def _tc_fwd_chosen(x, w, b, stride, padding) -> bool:
    """Did (or does, on first sight of this shape) the autotuner give this layer's forward convolution to the wgmma kernel?"""
    from . import tc_conv

    def lib():
        z = _conv(x, w, stride, padding)
        if not _nhwc(z):
            z = z.contiguous(memory_format=torch.channels_last)
        n, c, h, wd = z.shape
        _chk(_L().bnet_nn_bias_relu(z.data_ptr(), b.data_ptr(), n * h * wd, c, _DT[z.dtype], _stream()), "bias_relu")
        return z

    return tc_conv.choose("fwd", x, w, lib, lambda: tc_conv.conv3x3(x, w, b, relu=True), tc_conv.close) == "tc"


def _is_3x3_s1p1(w, stride, padding) -> bool:
    return tuple(w.shape[2:]) == (3, 3) and list(stride) == [1, 1] and list(padding) == [1, 1]


def _conv_bias_relu(x, w, b, stride, padding):
    """relu(conv(x, w) + b), NHWC: ONE wgmma kernel (bias + ReLU applied in the epilogue) where the autotuner picked it for this
    shape, otherwise cuDNN's convolution followed by our in-place bias + ReLU pass."""
    def lib():
        z = _conv(x, w, stride, padding)
        if not _nhwc(z):
            z = z.contiguous(memory_format=torch.channels_last)
        n, c, h, wd = z.shape
        _chk(_L().bnet_nn_bias_relu(z.data_ptr(), b.data_ptr(), n * h * wd, c, _DT[z.dtype], _stream()), "bias_relu")
        return z

    if _is_3x3_s1p1(w, stride, padding) and x.dtype == torch.bfloat16:
        from . import tc_conv

        def tc():
            return tc_conv.conv3x3(x, w, b, relu=True)

        if tc_conv.choose("fwd", x, w, lib, tc, tc_conv.close) == "tc":
            return tc()
    return lib()


class _ConvBiasReLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, stride, padding):
        z = _conv_bias_relu(x, w, b, stride, padding)
        ctx.save_for_backward(x, w, z)
        ctx.conv = (stride, padding)
        return z

    @staticmethod
    def backward(ctx, gy):
        x, w, y = ctx.saved_tensors
        stride, padding = ctx.conv
        if not _nhwc(gy):
            gy = gy.contiguous(memory_format=torch.channels_last)
        n, c, h, wd = y.shape
        gb = torch.zeros(c, device=y.device, dtype=torch.float32)
        gz = torch.empty_like(gy)
        _chk(_L().bnet_nn_relu_bwd_bias_grad(gy.data_ptr(), y.data_ptr(), gz.data_ptr(), gb.data_ptr(),
                                             _partials(c, y.device).data_ptr(), n * h * wd, c,
                                             _DT[y.dtype], _stream()), "relu_bwd_bias_grad")
        gx, gw = _conv_backward(gz, x, w, stride, padding, ctx.needs_input_grad[0])
        return gx, gw, gb.to(w.dtype), None, None


class _ConvBiasReLUPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, stride, padding):
        pool_bias = b
        if _is_3x3_s1p1(w, stride, padding) and x.dtype == torch.bfloat16 and _tc_fwd_chosen(x, w, b, stride, padding):
            # the wgmma convolution has bias + ReLU in its epilogue: the pool pass sees relu(z + b) and adds nothing
            from . import tc_conv

            z = tc_conv.conv3x3(x, w, b, relu=True)
            pool_bias = _zero_bias(b)
        else:
            z = _conv(x, w, stride, padding)
            if not _nhwc(z):
                z = z.contiguous(memory_format=torch.channels_last)
        n, c, h, wd = z.shape
        p = torch.empty((n, c, h // 2, wd // 2), device=z.device, dtype=z.dtype, memory_format=torch.channels_last)
        idx = torch.empty(n * (h // 2) * (wd // 2) * c, device=z.device, dtype=torch.uint8)
        _chk(_L().bnet_nn_bias_relu_pool_fwd(z.data_ptr(), pool_bias.data_ptr(), p.data_ptr(), idx.data_ptr(), n, h, wd, c,
                                             _DT[z.dtype], _stream()), "bias_relu_pool_fwd")
        ctx.save_for_backward(x, w, idx)
        ctx.conv = (stride, padding)
        ctx.zshape = (n, c, h, wd)
        return p

    @staticmethod
    def backward(ctx, gp):
        x, w, idx = ctx.saved_tensors
        stride, padding = ctx.conv
        n, c, h, wd = ctx.zshape
        if not _nhwc(gp):
            gp = gp.contiguous(memory_format=torch.channels_last)
        gb = torch.zeros(c, device=gp.device, dtype=torch.float32)
        gz = torch.empty((n, c, h, wd), device=gp.device, dtype=gp.dtype, memory_format=torch.channels_last)
        _chk(_L().bnet_nn_pool_relu_bwd_bias_grad(gp.data_ptr(), idx.data_ptr(), gz.data_ptr(), gb.data_ptr(),
                                                  _partials(c, gp.device).data_ptr(), n, h, wd, c,
                                                  _DT[gp.dtype], _stream()), "pool_relu_bwd_bias_grad")
        gx, gw = _conv_backward(gz, x, w, stride, padding, ctx.needs_input_grad[0])
        return gx, gw, gb.to(w.dtype), None, None


class _ConvBNAct(torch.autograd.Function):
    """y = relu?(batch_norm_train(conv(x, w)) (+ res)) — csrc/cuda/nn_kernels.cu, BatchNorm family."""

    @staticmethod
    def forward(ctx, x, w, gamma, beta, res, running_mean, running_var, stride, padding, eps, momentum, relu):
        z = _conv(x, w, stride, padding)
        if not _nhwc(z):
            z = z.contiguous(memory_format=torch.channels_last)
        n, c, h, wd = z.shape
        rows, dt, L = n * h * wd, _DT[z.dtype], _L()
        stats = torch.zeros(2 * c, device=z.device, dtype=torch.float32)
        _chk(L.bnet_nn_bn_stats(z.data_ptr(), stats.data_ptr(), _partials(2 * c, z.device).data_ptr(), rows, c, dt, _stream()),
             "bn_stats")
        if res is not None and not _nhwc(res):
            res = res.contiguous(memory_format=torch.channels_last)
        y = torch.empty_like(z)
        _chk(L.bnet_nn_bn_apply(z.data_ptr(), res.data_ptr() if res is not None else None, y.data_ptr(), stats.data_ptr(),
                                gamma.data_ptr(), beta.data_ptr(),
                                running_mean.data_ptr() if running_mean is not None else None,
                                running_var.data_ptr() if running_var is not None else None,
                                rows, c, eps, momentum, 1 if relu else 0, dt, _stream()), "bn_apply")
        ctx.save_for_backward(x, w, z, y, gamma, stats)
        ctx.cfg = (stride, padding, eps, relu, res is not None)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w, z, y, gamma, stats = ctx.saved_tensors
        stride, padding, eps, relu, has_res = ctx.cfg
        if not _nhwc(gy):
            gy = gy.contiguous(memory_format=torch.channels_last)
        n, c, h, wd = z.shape
        rows, dt, L = n * h * wd, _DT[z.dtype], _L()
        gsum = torch.zeros(2 * c, device=z.device, dtype=torch.float32)
        _chk(L.bnet_nn_bn_bwd_reduce(gy.data_ptr(), y.data_ptr(), z.data_ptr(), stats.data_ptr(), gsum.data_ptr(),
                                     _partials(2 * c, z.device).data_ptr(), rows, c, eps,
                                     1 if relu else 0, dt, _stream()), "bn_bwd_reduce")
        gz = torch.empty_like(z)
        gres = torch.empty_like(z) if has_res else None
        dgamma, dbeta = torch.empty_like(gamma), torch.empty_like(gamma)
        _chk(L.bnet_nn_bn_bwd_apply(gy.data_ptr(), y.data_ptr(), z.data_ptr(), gz.data_ptr(),
                                    gres.data_ptr() if has_res else None, stats.data_ptr(), gsum.data_ptr(), gamma.data_ptr(),
                                    dgamma.data_ptr(), dbeta.data_ptr(), rows, c, eps, 1 if relu else 0, dt, _stream()),
             "bn_bwd_apply")
        gx, gw = _conv_backward(gz, x, w, stride, padding, ctx.needs_input_grad[0])
        return gx, gw, dgamma, dbeta, gres, None, None, None, None, None, None, None


def conv_bn_act(x: torch.Tensor, conv: nn.Conv2d, bn: nn.BatchNorm2d, relu: bool = True, res: torch.Tensor | None = None):
    """relu?(bn(conv(x)) (+ res)) for one ResNet stage.  Training mode with channels_last bf16/fp32 tensors runs the fused
    kernels (statistics, normalise + affine + residual + ReLU in one pass, two-kernel backward); anything else
    (eval mode, exotic configurations) takes the eager PyTorch chain."""
    c = conv.out_channels
    vec = 8 if x.dtype == torch.bfloat16 else 4
    if (bn.training and _supported(x, c) and c // vec <= 256 and conv.bias is None and conv.groups == 1
            and conv.dilation == (1, 1) and bn.affine and bn.track_running_stats and bn.momentum is not None
            and bn.weight.dtype == x.dtype and bn.running_mean.dtype == x.dtype):
        if not _nhwc(x):
            x = x.contiguous(memory_format=torch.channels_last)
        if bn.num_batches_tracked is not None:
            bn.num_batches_tracked.add_(1)
        return _ConvBNAct.apply(x, conv.weight, bn.weight, bn.bias, res, bn.running_mean, bn.running_var,
                                list(conv.stride), list(conv.padding), float(bn.eps), float(bn.momentum), bool(relu))
    y = bn(conv(x))
    if res is not None:
        y = y + res
    return torch.relu(y) if relu else y


def self_check(device=None, verbose: bool = False) -> bool:
    """One small fused block (with and without pooling), forward and backward, against the eager PyTorch chain in
    bf16.  Cheap (a few ms); lets a training script fall back to eager layers instead of training on wrong
    gradients if the native kernels misbehave on this machine."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else device
    try:
        g = torch.Generator(device=dev).manual_seed(1234)
        # narrow and wide channel counts (8 and 64 16-byte channel groups per pixel), with and without pooling
        # ... and two layers at the benchmark's own spatial sizes (millions of rows: the capped, grid-striding launch)
        for cin, cout, hw, pool in ((16, 64, 20, False), (16, 64, 20, True), (32, 512, 14, False), (32, 512, 14, True),
                                    (16, 64, 224, True), (32, 128, 112, False)):
            blk = ConvBiasReLU(cin, cout, 3, 1, 1, pool=pool).to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
            x = torch.randn(3, cin, hw, hw, device=dev, generator=g).to(torch.bfloat16).contiguous(
                memory_format=torch.channels_last)
            xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
            ya = blk(xa)
            yb = torch.relu(blk.conv(xb))
            if pool:
                yb = nn.functional.max_pool2d(yb, 2, 2)
            go = torch.randn(yb.shape, device=dev, generator=g).to(torch.bfloat16)
            ya.backward(go)
            ga = [xa.grad.float().clone(), blk.conv.weight.grad.float().clone(), blk.conv.bias.grad.float().clone()]
            blk.zero_grad(set_to_none=True)
            yb.backward(go)
            gb = [xb.grad.float(), blk.conv.weight.grad.float(), blk.conv.bias.grad.float()]
            torch.cuda.synchronize(dev)
            errs = [((ya.float() - yb.float()).norm() / yb.float().norm().clamp_min(1e-6)).item()]
            errs += [((a - b).norm() / b.norm().clamp_min(1e-6)).item() for a, b in zip(ga, gb)]
            if verbose:
                print(f"[fused_nn.self_check] {cin}->{cout} {hw}x{hw} pool={pool} relative L2 errors (y, gx, gw, gb): {errs}")
            # (bf16 near-ties route a few pool / ReLU gradients differently than the eager chain: a real indexing bug
            #  shows up as an error of order 1, not of order 0.01)
            if not all(e == e and e < 0.15 for e in errs):
                return False
        return True
    except Exception as e:      # noqa: BLE001 - any failure means "do not use the fused path"
        if verbose:
            print(f"[fused_nn.self_check] failed: {e!r}")
        return False


def self_check_bn(device=None, verbose: bool = False) -> bool:
    """The BatchNorm family (conv_bn_act) against the eager chain, bf16, forward / backward / running statistics."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else device
    try:
        g = torch.Generator(device=dev).manual_seed(4321)
        for cin, cout, hw, k, relu, with_res in ((16, 64, 14, 3, True, False), (64, 256, 8, 1, True, True), (32, 2048, 4, 1, False, False)):
            conv = nn.Conv2d(cin, cout, k, 1, k // 2, bias=False).to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
            bn_a = nn.BatchNorm2d(cout).to(dev).to(torch.bfloat16)
            with torch.no_grad():
                bn_a.weight.copy_(torch.rand(cout, device=dev, generator=g) + 0.5)
                bn_a.bias.copy_(torch.randn(cout, device=dev, generator=g) * 0.1)
            import copy

            bn_b = copy.deepcopy(bn_a)
            x = torch.randn(4, cin, hw, hw, device=dev, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
            res = torch.randn(4, cout, hw, hw, device=dev, generator=g).to(torch.bfloat16).contiguous(
                memory_format=torch.channels_last) if with_res else None
            xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
            ra = res.clone().requires_grad_(True) if with_res else None
            rb = res.clone().requires_grad_(True) if with_res else None
            ya = conv_bn_act(xa, conv, bn_a, relu=relu, res=ra)
            go = torch.randn(ya.shape, device=dev, generator=g).to(torch.bfloat16)
            ya.backward(go)
            ga = [xa.grad.float().clone(), conv.weight.grad.float().clone(), bn_a.weight.grad.float().clone(), bn_a.bias.grad.float().clone()]
            if with_res:
                ga.append(ra.grad.float().clone())
            conv.zero_grad(set_to_none=True)
            yb = bn_b(conv(xb))
            if with_res:
                yb = yb + rb
            if relu:
                yb = torch.relu(yb)
            yb.backward(go)
            gb = [xb.grad.float(), conv.weight.grad.float(), bn_b.weight.grad.float(), bn_b.bias.grad.float()]
            if with_res:
                gb.append(rb.grad.float())
            torch.cuda.synchronize(dev)
            rel = lambda a, b: ((a - b).norm() / b.norm().clamp_min(1e-6)).item()      # noqa: E731
            errs = [rel(ya.float(), yb.float())] + [rel(a, b) for a, b in zip(ga, gb)]
            errs += [rel(bn_a.running_mean.float(), bn_b.running_mean.float()), rel(bn_a.running_var.float(), bn_b.running_var.float())]
            if verbose:
                print(f"[fused_nn.self_check_bn] {cin}->{cout} k{k} {hw}x{hw} relu={relu} res={with_res} relative L2 errors: {errs}")
            if not all(e == e and e < 0.15 for e in errs):
                return False
            if int(bn_a.num_batches_tracked.item()) != 1:
                return False
        return True
    except Exception as e:      # noqa: BLE001
        if verbose:
            print(f"[fused_nn.self_check_bn] failed: {e!r}")
        return False


class ConvBiasReLU(nn.Module):
    """3x3 (or any) convolution + bias + ReLU, optionally followed by a 2x2/stride-2 max-pool."""

    def __init__(self, cin: int, cout: int, kernel_size: int = 3, stride: int = 1, padding: int = 1, pool: bool = False):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, kernel_size, stride, padding)
        self.pool = pool

    @property
    def weight(self):
        return self.conv.weight

    @property
    def bias(self):
        return self.conv.bias

    def forward(self, x):
        c = self.conv
        k, s_, p_ = c.kernel_size, c.stride, c.padding
        ho = (x.shape[2] + 2 * p_[0] - k[0]) // s_[0] + 1
        wo = (x.shape[3] + 2 * p_[1] - k[1]) // s_[1] + 1
        if _supported(x, c.out_channels) and c.groups == 1 and c.dilation == (1, 1) and (
                not self.pool or (ho % 2 == 0 and wo % 2 == 0)):
            if not _nhwc(x):
                x = x.contiguous(memory_format=torch.channels_last)
            fn = _ConvBiasReLUPool if self.pool else _ConvBiasReLU
            return fn.apply(x, c.weight, c.bias, list(c.stride), list(c.padding))
        y = torch.relu(c(x))
        return nn.functional.max_pool2d(y, 2, 2) if self.pool else y

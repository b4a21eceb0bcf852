"""3x3 convolution on the wgmma tensor cores (csrc/cuda/tc_gemm.cu, ``kConv`` instantiations).

    y  = tc_conv.conv3x3(x, w, bias, relu=True)     # NHWC bf16, stride 1, pad 1; bias + ReLU applied in the epilogue
    dx = tc_conv.conv3x3_dgrad(gy, w)               # same filter, read MN-major with flipped taps (no rotated copy)
    dw = tc_conv.conv3x3_wgrad(gy, x)               # filter gradient: the reduction runs over 64-pixel TMA boxes of gy and x

Implicit GEMM: the 128 accumulator rows of a tile are a patch of output pixels (bw x bh pixels of bn images); for every
(filter tap, 64-channel block) the patch's shifted input arrives as ONE 4-D TMA box of the NHWC activation, the padding
being the TMA unit's zero fill.  No im2col buffer exists anywhere.  Filters are used exactly as torch stores a
channels_last ``Conv2d.weight`` ([Cout][3][3][Cin]).

The filter gradient ``dw[co, tap, ci] = sum_p gy[p, co] * x[p + tap, ci]`` is the same kernel with both operands MN-major
(the layout the linear layer's ``dW = gY^T . X`` uses): 64-pixel boxes of ``gy`` ride the accumulator rows, 64-pixel boxes of the
shifted ``x`` the columns, the pixel blocks are split over ``grid.z`` and the slice that arrives last at a tile converts
the fp32 sums to bf16 — the result is the ``channels_last`` weight gradient itself.  ``wgrad_trusted()`` lets it run only
after ``self_check_wgrad()`` passed in a CHILD process on this GPU
(verdict cached per library build and GPU model; ``BNET_TC_WGRAD=0`` disables it, ``=1`` skips the child).

The layers above (``fused_nn.ConvBiasReLU``) ask ``choose()`` which implementation to run for a given shape: on first
(eager) use each candidate is timed on the actual tensors with CUDA events and the winner is cached for the process (our
kernel wins only by a clear margin, ``TC_MARGIN``) —
so a shape where cuDNN's kernel is faster keeps cuDNN.  ``BNET_TC_CONV=1`` forces the wgmma kernels wherever the
shape allows, ``=0`` disables them, default ``auto``.

The reference has no compute path (SURVEY.md section 2.6); this is part of the GPU training engine around the transport."""
from __future__ import annotations

import ctypes as C
import os

import torch

from ..utils.native import load
from . import tc_linear

_lib = None
LAUNCHES = 0
_choice: dict = {}          # (kind, N, H, W, Cin, Cout) -> "tc" | "cudnn"
TIMINGS: dict = {}          # the same key -> {"tc": us, "cudnn": us}  (what the autotuner measured; bench.py reports it)


def _L():
    global _lib
    if _lib is None:
        _lib = load()
        vp, i = C.c_void_p, C.c_int
        _lib.bnet_tc_conv3x3.argtypes = [vp, vp, vp, vp, i, i, i, i, i, i, vp, vp]
        _lib.bnet_tc_conv3x3_dgrad.argtypes = [vp, vp, vp, i, i, i, i, i, vp, vp]
        _lib.bnet_tc_conv3x3_wgrad.argtypes = [vp, vp, vp, vp, vp, i, i, i, i, i, i, vp, vp]
        _lib.bnet_tc_conv3x3_wgrad_tiles.argtypes = [i, i]
        _lib.bnet_tc_conv3x3_wgrad_plan.argtypes = [i, i, i, i, i, i, C.POINTER(tc_linear.Plan)]
        _lib.bnet_tc_last_error.restype = C.c_char_p
    return _lib


def mode() -> str:
    v = os.environ.get("BNET_TC_CONV", "auto").lower()
    return {"1": "on", "0": "off", "on": "on", "off": "off"}.get(v, "auto")


def _nhwc(t: torch.Tensor) -> bool:
    return t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last)


def shape_ok(x: torch.Tensor, w: torch.Tensor, dgrad: bool = False) -> bool:
    """3x3 / stride 1 / pad 1 is checked by the caller; here: dtype, layout and the kernel's channel constraints."""
    if not (x.is_cuda and x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 and _nhwc(x)):
        return False
    cout, cin = w.shape[0], w.shape[1]
    if tuple(w.shape[2:]) != (3, 3) or not w.is_contiguous(memory_format=torch.channels_last):
        return False
    if w.data_ptr() % 16 or x.data_ptr() % 16:
        return False
    if dgrad:
        return cout % 64 == 0 and cin % 64 == 0
    return cin % 64 == 0 and cout % 8 == 0


def usable() -> bool:
    return mode() != "off" and tc_linear.supported() and tc_linear.trusted()


def conv3x3(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None, relu: bool = False,
            out: torch.Tensor | None = None) -> torch.Tensor:
    """relu?(conv2d(x, w, bias, stride=1, padding=1)) — x [N,Cin,H,W] channels_last, w [Cout,Cin,3,3] channels_last, bf16."""
    global LAUNCHES
    n, cin, h, wd = x.shape
    cout = w.shape[0]
    if out is None:
        out = torch.empty((n, cout, h, wd), device=x.device, dtype=torch.bfloat16, memory_format=torch.channels_last)
    L = _L()
    rc = L.bnet_tc_conv3x3(x.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None, out.data_ptr(), n, h, wd, cin,
                           cout, 1 if relu else 0, tc_linear._err_flag(x.device.index).data_ptr(), tc_linear._stream())
    if rc < 0:
        raise RuntimeError(f"bnet_tc_conv3x3: {L.bnet_tc_last_error().decode()}")
    LAUNCHES += rc
    tc_linear.LAUNCHES += rc
    return out


def conv3x3_dgrad(gy: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """Input gradient of the same convolution: gy [N,Cout,H,W] channels_last -> dx [N,Cin,H,W] channels_last."""
    global LAUNCHES
    n, cout, h, wd = gy.shape
    cin = w.shape[1]
    dx = torch.empty((n, cin, h, wd), device=gy.device, dtype=torch.bfloat16, memory_format=torch.channels_last)
    L = _L()
    rc = L.bnet_tc_conv3x3_dgrad(gy.data_ptr(), w.data_ptr(), dx.data_ptr(), n, h, wd, cin, cout,
                                 tc_linear._err_flag(gy.device.index).data_ptr(), tc_linear._stream())
    if rc < 0:
        raise RuntimeError(f"bnet_tc_conv3x3_dgrad: {L.bnet_tc_last_error().decode()}")
    LAUNCHES += rc
    tc_linear.LAUNCHES += rc
    return dx


def wgrad_plan(n: int, h: int, w: int, cin: int, cout: int, splits: int = 0) -> dict:
    """The tiling the filter-gradient kernel would use (host-only; works without a GPU)."""
    p = tc_linear.Plan()
    if _L().bnet_tc_conv3x3_wgrad_plan(n, h, w, cin, cout, splits, C.byref(p)) != 0:
        raise ValueError(_L().bnet_tc_last_error().decode())
    return p.as_dict()


_wgrad_scratch: dict = {}


def _wgrad_ws(device, cin: int, cout: int):
    """fp32 [Cout, 9 Cin] workspace + tile counters of the split-K fix-up, shared by every call of that shape on that device
    (calls on one stream are ordered; the kernel hands both back all-zero)."""
    key = (device.index, cin, cout)
    if key not in _wgrad_scratch:
        tiles = _L().bnet_tc_conv3x3_wgrad_tiles(cin, cout)
        _wgrad_scratch[key] = (torch.zeros((cout, 9 * cin), dtype=torch.float32, device=device),
                               torch.zeros(tiles + 8, dtype=torch.int32, device=device))
    return _wgrad_scratch[key]


def wgrad_shape_ok(gy: torch.Tensor, x: torch.Tensor) -> bool:
    if not (gy.is_cuda and gy.dtype == torch.bfloat16 and x.dtype == torch.bfloat16 and _nhwc(gy) and _nhwc(x)):
        return False
    if gy.shape[0] != x.shape[0] or gy.shape[2:] != x.shape[2:] or gy.data_ptr() % 16 or x.data_ptr() % 16:
        return False
    return gy.shape[1] % 64 == 0 and x.shape[1] % 64 == 0


def conv3x3_wgrad(gy: torch.Tensor, x: torch.Tensor, splits: int = 0, out: torch.Tensor | None = None) -> torch.Tensor:
    """Filter gradient of ``conv2d(x, w, stride=1, padding=1)``: gy [N,Cout,H,W], x [N,Cin,H,W] channels_last bf16 ->
    dw [Cout,Cin,3,3] channels_last bf16 (memory [Cout][3][3][Cin]).  ``splits``: slices of the pixel reduction (0 = as many
    as fill the SMs)."""
    global LAUNCHES
    n, cout, h, wd = gy.shape
    cin = x.shape[1]
    # `out`: a channels_last bf16 [Cout,Cin,3,3] tensor to write into (the parameter's slice of an engine's flat gradient buffer)
    if out is not None and (tuple(out.shape) != (cout, cin, 3, 3) or out.dtype != torch.bfloat16 or out.data_ptr() % 16
                            or not out.is_contiguous(memory_format=torch.channels_last)):
        out = None
    dw = out if out is not None else torch.empty((cout, cin, 3, 3), device=gy.device, dtype=torch.bfloat16,
                                                  memory_format=torch.channels_last)
    ws, counters = _wgrad_ws(gy.device, cin, cout)
    L = _L()
    rc = L.bnet_tc_conv3x3_wgrad(gy.data_ptr(), x.data_ptr(), dw.data_ptr(), ws.data_ptr(), counters.data_ptr(), n, h, wd, cin, cout,
                                 splits, tc_linear._err_flag(gy.device.index).data_ptr(), tc_linear._stream())
    if rc < 0:
        raise RuntimeError(f"bnet_tc_conv3x3_wgrad: {L.bnet_tc_last_error().decode()}")
    if os.environ.get("BNET_TC_WGRAD_FIXUP", "1") == "0":
        # fall-back mode (the self-check's ladder): the kernel only added its slices' sums into the fp32 workspace
        dw.copy_(ws.view(cout, 3, 3, cin).permute(0, 3, 1, 2))
        ws.zero_()
    LAUNCHES += rc
    tc_linear.LAUNCHES += rc
    return dw


_wgrad_trusted = None


def _extra_check_shapes():
    """(tuple of (n, cin, cout, hw, 0) from BNET_TC_WGRAD_CHECK_SHAPES, suffix for the verdict's cache file)."""
    import hashlib

    raw = os.environ.get("BNET_TC_WGRAD_CHECK_SHAPES", "").strip()
    shapes = []
    for item in raw.split(";"):
        try:
            n, cin, cout, hw = (int(v) for v in item.split(","))
        except ValueError:
            continue
        if n > 0 and hw > 0 and cin % 64 == 0 and cout % 64 == 0 and cin > 0 and cout > 0:
            shapes.append((n, cin, cout, hw, 0))
    shapes = tuple(sorted(set(shapes)))
    return shapes, ("_" + hashlib.sha1(repr(shapes).encode()).hexdigest()[:8]) if shapes else ""


def wgrad_trusted() -> bool:
    """May the filter-gradient kernel run in THIS process?  ``BNET_TC_WGRAD``: ``0`` never, ``1`` yes (no check), default:
    only after ``self_check_wgrad()`` passed in a child process on this GPU — a kernel that faults there must not be able
    to poison the training process' CUDA context.  The verdict is cached per library build and GPU model."""
    global _wgrad_trusted
    if _wgrad_trusted is None:
        v = os.environ.get("BNET_TC_WGRAD", "auto").lower()
        if v in ("0", "off") or not usable():
            _wgrad_trusted = False
        elif v in ("1", "on"):
            _wgrad_trusted = True
        else:
            if torch.cuda.is_current_stream_capturing():
                return False
            # BNET_TC_WGRAD_CHECK_SHAPES="n,cin,cout,hw;...": layer shapes the caller is about to train (bench.py names the
            # flagship's) are checked in the child as well, so that a shape-dependent fault cannot happen in this process
            extra, sfx = _extra_check_shapes()
            check = f"from bagua_net_b200.ops import tc_conv; ok = tc_conv.self_check_wgrad(shapes=tc_conv.WGRAD_CHECK_SHAPES + {extra!r})"
            # Fallback ladder.  Two building blocks of this kernel are shared with no hardware-validated kernel: the 256-column
            # MN-major column operand (the linear dW ran 128-column tiles) and the in-kernel finish of the split reduction in
            # this orientation (the linear layer's ran with swapped operands).  If the default configuration fails its check,
            # the configurations without one or both of them are tried; the library reads the variables at its first
            # filter-gradient launch, which cannot have happened yet in this process.
            ladder = ({}, {"BNET_TC_WGRAD_BN": "128"}, {"BNET_TC_WGRAD_FIXUP": "0"}, {"BNET_TC_WGRAD_BN": "128", "BNET_TC_WGRAD_FIXUP": "0"})
            preset = any(k in os.environ for k in ("BNET_TC_WGRAD_BN", "BNET_TC_WGRAD_FIXUP"))
            _wgrad_trusted = False
            # the whole ladder is bounded in time (BNET_TC_WGRAD_BUDGET_S, default 240 s: every rung is a fresh process that
            # imports torch on a possibly cold machine); a rung that cannot start within what is left is not tried
            import time

            budget = float(os.environ.get("BNET_TC_WGRAD_BUDGET_S", "240") or 240)
            t_start = time.monotonic()
            for cfg in (ladder[:1] if preset else ladder):
                left = budget - (time.monotonic() - t_start)
                if left < 20.0:
                    break
                os.environ.update(cfg)
                tag = ("tc_wgrad" + ("_bn128" if os.environ.get("BNET_TC_WGRAD_BN") == "128" else "")
                       + ("_nofix" if os.environ.get("BNET_TC_WGRAD_FIXUP") == "0" else ""))
                if tc_linear._isolated_self_check(timeout=min(180.0, left), check=check, tag=tag + "_self_check" + sfx):
                    _wgrad_trusted = True
                    break
                for k in cfg:
                    os.environ.pop(k, None)
                if not tc_linear.LAST_CHECK_DEFINITIVE:
                    break       # the child could not run or timed out: the next rung would wait just as long for nothing
    return _wgrad_trusted


def prepare() -> dict:
    """Settle every once-per-process verdict NOW: the linear / convolution kernels' self-check and the filter gradient's
    child-process check (tens of seconds the first time on a machine, a file read afterwards).  Training engines call this
    before their first collective, so that no rank sits in a child process while its peers already wait inside one —
    the cross-rank barriers of the fused kernels carry a 20 s watchdog."""
    if not torch.cuda.is_available() or torch.cuda.is_current_stream_capturing():
        return {"usable": False, "wgrad": False}
    u = usable()
    return {"usable": u, "wgrad": wgrad_trusted() if u else False}


def choose_wgrad(gy: torch.Tensor, x: torch.Tensor, w: torch.Tensor, cudnn_fn) -> str:
    """"tc" or "cudnn" for this layer's filter gradient: like ``choose`` (results compared, both timed, winner cached per
    shape), behind ``wgrad_trusted()``."""
    n, cout, h, wd = gy.shape
    key = ("wgrad", n, h, wd, x.shape[1], cout)
    got = _choice.get(key)
    if got is not None:
        return got
    m = mode()
    if m == "off" or not usable() or not wgrad_shape_ok(gy, x) or not w.is_contiguous(memory_format=torch.channels_last):
        _choice[key] = "cudnn"
        return "cudnn"
    if torch.cuda.is_current_stream_capturing():
        return "cudnn"
    if not wgrad_trusted():
        _choice[key] = "cudnn"
        TIMINGS[key] = {"error": "weight-gradient kernel not trusted on this GPU (self-check in a child process failed or BNET_TC_WGRAD=0)"}
        return "cudnn"
    try:
        def tc_fn():
            return conv3x3_wgrad(gy, x)

        a, b = tc_fn(), cudnn_fn()
        torch.cuda.synchronize()
        if tc_linear.last_error(gy.device.index):
            raise RuntimeError("pipeline watchdog")
        if not close(a, b):
            raise RuntimeError("results differ from cuDNN")
        del a, b
        if m == "on":
            _choice[key] = "tc"
            return "tc"
        t_tc, t_cudnn = _time_us(tc_fn), _time_us(cudnn_fn)
        TIMINGS[key] = {"tc": round(t_tc, 1), "cudnn": round(t_cudnn, 1)}
        _choice[key] = _faster(t_tc, t_cudnn)
    except Exception as ex:   # noqa: BLE001 — anything unexpected keeps the library path for this shape
        TIMINGS[key] = {"error": f"{type(ex).__name__}: {str(ex)[:80]}"}
        _choice[key] = "cudnn"
        try:        # a run that went wrong may have left the shared scratch of this (Cin, Cout) dirty: other shapes use it too
            ws, counters = _wgrad_ws(gy.device, x.shape[1], cout)
            ws.zero_()
            counters.zero_()
        except Exception:   # noqa: BLE001
            pass
    return _choice[key]


# Our kernel replaces cuDNN only when it is clearly faster: the two round differently, so a choice that followed timing noise
# on a near-tie would make the same program compute different numbers from run to run.
TC_MARGIN = 0.9


def _faster(t_tc: float, t_cudnn: float) -> str:
    return "tc" if t_tc <= TC_MARGIN * t_cudnn else "cudnn"


def _time_us(fn, iters: int = 5) -> float:
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def choose(kind: str, x: torch.Tensor, w: torch.Tensor, cudnn_fn, tc_fn, check=None) -> str:
    """Which implementation runs this (kind, shape): decided once per process by timing both on the actual tensors (never
    inside a CUDA-graph capture: an undecided shape keeps cuDNN there), after comparing their results (`check(a, b)`)."""
    n, c, h, wd = x.shape
    key = (kind, n, h, wd, w.shape[1], w.shape[0])
    got = _choice.get(key)
    if got is not None:
        return got
    m = mode()
    if m == "off" or not usable() or not shape_ok(x, w, dgrad=(kind == "dgrad")):
        _choice[key] = "cudnn"
        return "cudnn"
    if torch.cuda.is_current_stream_capturing():
        return "tc" if m == "on" else "cudnn"
    try:
        a, b = tc_fn(), cudnn_fn()
        torch.cuda.synchronize()
        if tc_linear.last_error(x.device.index):
            raise RuntimeError("pipeline watchdog")
        if check is not None and not check(a, b):
            raise RuntimeError("results differ from cuDNN")
        del a, b
        if m == "on":
            _choice[key] = "tc"
            return "tc"
        t_tc, t_cudnn = _time_us(tc_fn), _time_us(cudnn_fn)
        TIMINGS[key] = {"tc": round(t_tc, 1), "cudnn": round(t_cudnn, 1)}
        _choice[key] = _faster(t_tc, t_cudnn)
    except Exception as ex:   # noqa: BLE001 — anything unexpected keeps the library path for this shape
        TIMINGS[key] = {"error": f"{type(ex).__name__}: {str(ex)[:80]}"}
        _choice[key] = "cudnn"
    return _choice[key]


def close(a: torch.Tensor, b: torch.Tensor) -> bool:
    d = (a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-6)
    return bool(d == d and d < 2e-2)


def self_check(device=None, verbose: bool = False) -> bool:
    """Forward and input-gradient kernels against cuDNN in bf16: exact patches, ragged ones, several images per patch."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else device
    g = torch.Generator(device=dev).manual_seed(99)
    ok = True
    for n, cin, cout, hw in ((2, 64, 64, 32), (3, 64, 128, 14), (2, 128, 256, 28), (5, 256, 64, 7), (1, 64, 320, 20)):
        x = torch.randn(n, cin, hw, hw, device=dev, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        w = (torch.randn(cout, cin, 3, 3, device=dev, generator=g) * (1.0 / (3 * cin ** 0.5))).to(torch.bfloat16).contiguous(
            memory_format=torch.channels_last)
        b = torch.randn(cout, device=dev, generator=g).to(torch.bfloat16)
        y = conv3x3(x, w, b, relu=True)
        ref = torch.relu(torch.nn.functional.conv2d(x, w, b, 1, 1))
        e1 = ((y.float() - ref.float()).norm() / ref.float().norm()).item()
        errs = [e1]
        if cout % 64 == 0:
            gy = torch.randn(n, cout, hw, hw, device=dev, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
            dx = conv3x3_dgrad(gy, w)
            dref = torch.ops.aten.convolution_backward(gy, x, w, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [True, False, False])[0]
            errs.append(((dx.float() - dref.float()).norm() / dref.float().norm()).item())
        torch.cuda.synchronize()
        bad = tc_linear.last_error(dev.index)
        if verbose:
            print(f"[tc_conv.self_check] N={n} {cin}->{cout} {hw}x{hw}: relative L2 errors {errs} watchdog {bad}")
        ok = ok and bad == 0 and all(e == e and e < 2e-2 for e in errs)
    return ok


WGRAD_CHECK_SHAPES = ((2, 64, 64, 32, 0), (3, 64, 128, 14, 1), (2, 128, 256, 28, 0), (5, 256, 64, 7, 3), (1, 64, 320, 20, 0),
                      (32, 512, 512, 14, 0), (8, 128, 128, 56, 0))       # (batch, Cin, Cout, height = width, pixel slices)


def self_check_wgrad(device=None, verbose: bool = False, shapes=WGRAD_CHECK_SHAPES) -> bool:
    """The filter-gradient kernel against cuDNN in bf16: exact and ragged 64-pixel patches, one and many slices of the pixel
    reduction, Cout below one lane tile, tiles that straddle taps (Cin = 64), columns past 9 Cin (Cin = 128), a VGG-sized
    layer; the workspace and the tile counters must come back all zero."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else device
    g = torch.Generator(device=dev).manual_seed(7)
    ok = True
    for n, cin, cout, hw, splits in shapes:
        x = torch.randn(n, cin, hw, hw, device=dev, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        gy = (torch.randn(n, cout, hw, hw, device=dev, generator=g) * (1.0 / hw)).to(torch.bfloat16).contiguous(
            memory_format=torch.channels_last)
        w = torch.empty(cout, cin, 3, 3, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
        errs = []
        for _ in range(2):                    # twice: the second call runs on the scratch the first one handed back
            dw = conv3x3_wgrad(gy, x, splits)
            ref = torch.ops.aten.convolution_backward(gy, x, w, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [False, True, False])[1]
            errs.append(((dw.float() - ref.float()).norm() / ref.float().norm().clamp_min(1e-6)).item())
        torch.cuda.synchronize()
        bad = tc_linear.last_error(dev.index)
        ws, counters = _wgrad_ws(dev, cin, cout)
        clean = bool((ws == 0).all().item()) and bool((counters == 0).all().item())
        if verbose:
            print(f"[tc_conv.self_check_wgrad] N={n} {cin}->{cout} {hw}x{hw} splits={splits}: relative L2 errors {errs} watchdog {bad} "
                  f"scratch clean {clean}")
        ok = ok and bad == 0 and clean and all(e == e and e < 2e-2 for e in errs)
    return ok

"""Numerics of the wgmma linear / convolution kernels (csrc/cuda/tc_gemm.cu) and of the fused layers' NaN handling, run by
tests/test_tc_numerics.py one job per child process (a kernel fault must not poison the pytest process).

Every case is checked twice against the same operation in float64, computed from the very bf16 operands the kernel read:
- exact: sparse small-integer operands with every reference output |r| <= 256, so every fp32 partial sum is exact in any
  order and bf16 holds the result: the kernel's output must equal the reference rounded to bf16, bit for bit.  A dropped
  or repeated k-block, a wrong tap, pixel, column, bias entry or ReLU cannot hide behind a tolerance.
- bounded: Gaussian operands, |y - r| <= 2^-8 |r| + 2^-16 S with S = sum |a b| (+ |bias|): bf16 output rounding plus fp32
  accumulation.  Catches precision losses integers cannot show (a partial sum rounded to bf16, say).

The case list is chosen so that it reaches every one of the 22 kernel instantiations `(entry point, BN, swap)` the host
dispatch tables launch, each tile width at least once in persistent form (several tiles per CTA, the shared-memory ring
and the mbarrier parities wrapping more than once), plus the tilings the VGG16 batch-32 benchmark plans.  `coverage`
checks that from the planners themselves (tc_linear.plan, tc_conv.conv_plan, tc_conv.wgrad_plan).

    python tests/tc_numerics_worker.py <job>          jobs: coverage linear conv vgg nan reductions
"""
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bagua_net_b200.ops import fused_nn, tc_conv, tc_linear  # noqa: E402

# every instantiation run(), run_conv() and run_conv_wgrad() dispatch to: (entry point, BN, swap)
EXPECTED = ({("linear", bn, int(bn < 128)) for bn in (32, 64, 128, 256)}
            | {("linear_splitk", bn, int(bn < 128)) for bn in (32, 64, 128, 256)}
            | {("linear_dgrad", bn, int(bn < 128)) for bn in (32, 64, 128, 256)}
            | {("linear_wgrad", 128, 0), ("linear_wgrad", 256, 0)}
            | {("conv", bn, 0) for bn in (64, 128, 256)} | {("conv_dgrad", bn, 0) for bn in (64, 128, 256)}
            | {("conv_wgrad", 128, 0), ("conv_wgrad", 256, 0)})


def L(op, M, N, K, relu=False, bias=True, splits=1, pad=0, name=""):
    """linear family: op = linear (x[M,K] w[N,K] -> [M,N]; splits None = automatic), dgrad (gy[M,N] w[N,K] -> [M,K]),
    wgrad (gy[M,N] x[M,K] -> [N,K]).  pad > 0: the output is a guarded view (row pitch + pad, or a slice of a flat buffer)."""
    return dict(op=op, M=M, N=N, K=K, relu=relu, bias=bias, splits=splits, pad=pad, name=name)


def CV(op, n, h, w, cin, cout, relu=False, bias=True, splits=0, pad=0, name=""):
    """convolution family: op = conv, conv_dgrad, conv_wgrad (splits: pixel slices, 0 = automatic)."""
    return dict(op=op, n=n, h=h, w=w, cin=cin, cout=cout, relu=relu, bias=bias, splits=splits, pad=pad, name=name)


LINEAR_CASES = [
    # forward: the swap / BN switch points M = 1, 32, 33, 64, 65; partial last k-block; odd N and N % 16 != 0 (scalar stores)
    L("linear", 1, 136, 200, relu=True), L("linear", 32, 131, 264, pad=24), L("linear", 33, 200, 72, relu=True),
    L("linear", 64, 520, 136), L("linear", 65, 131, 200, relu=True, pad=8), L("linear", 300, 1000, 1000, relu=True),
    # forward, many tiles per CTA (400 tiles on 132 CTAs, 8 k-blocks each)
    L("linear", 32, 51200, 512, relu=True), L("linear", 64, 51200, 512),
    L("linear", 2048, 4096, 512, relu=True, pad=8),
    # split-K: 2, 3, 8 and automatic slices, more slices than k-blocks, every tile width, several tiles per CTA
    L("linear", 32, 4096, 4096, relu=True, splits=None), L("linear", 48, 1000, 2048, splits=3, pad=16),
    L("linear", 17, 136, 128, relu=True, splits=8), L("linear", 64, 1000, 4096, splits=2),
    L("linear", 200, 520, 1000, relu=True, splits=3), L("linear", 256, 3072, 2048, splits=8),
    L("linear", 1024, 6400, 1024, relu=True, splits=2),
    L("linear", 32, 32768, 2048, splits=2), L("linear", 64, 32768, 2048, relu=True, splits=2),
    # dX: both orientations, several tiles per CTA
    L("dgrad", 1, 136, 264), L("dgrad", 33, 72, 200), L("dgrad", 65, 200, 520), L("dgrad", 300, 520, 136),
    L("dgrad", 32, 512, 51200), L("dgrad", 64, 512, 51200),
    L("dgrad", 512, 512, 25600),
    # dW: reduction over the batch, ragged batch (partial k-block), into a slice of a flat buffer
    L("wgrad", 33, 136, 264, pad=64), L("wgrad", 65, 200, 72), L("wgrad", 300, 520, 136, pad=64),
    L("wgrad", 64, 4096, 4096),
]

CONV_CASES = [
    # H != W, H and W not multiples of the patch, N not a multiple of its image count, Cin = 64, Cout = 8 * odd
    CV("conv", 3, 10, 22, 64, 72, relu=True), CV("conv", 5, 7, 9, 128, 40), CV("conv", 2, 30, 14, 64, 128, relu=True, pad=64),
    CV("conv", 3, 13, 6, 192, 200, relu=True), CV("conv", 1, 20, 12, 64, 320),
    CV("conv", 9, 28, 20, 64, 512, relu=True, pad=64),
    CV("conv", 6, 60, 40, 64, 64, relu=True), CV("conv", 4, 48, 40, 128, 128),
    CV("conv", 6, 36, 28, 128, 256, relu=True),
    CV("conv_dgrad", 3, 10, 22, 64, 64), CV("conv_dgrad", 5, 7, 9, 128, 64), CV("conv_dgrad", 2, 30, 14, 64, 128),
    CV("conv_dgrad", 9, 28, 20, 512, 256),
    CV("conv_dgrad", 6, 60, 40, 64, 64), CV("conv_dgrad", 4, 48, 40, 128, 128),
    CV("conv_dgrad", 6, 36, 28, 256, 256),
    # filter gradient: 1, several and automatic pixel slices, Cin = 64 (tiles straddle taps), several tiles per CTA
    CV("conv_wgrad", 3, 10, 22, 64, 64, splits=1), CV("conv_wgrad", 5, 7, 9, 128, 64, splits=3, pad=64),
    CV("conv_wgrad", 2, 30, 14, 64, 128), CV("conv_wgrad", 3, 13, 6, 192, 128, splits=0, pad=64),
    CV("conv_wgrad", 2, 32, 32, 64, 1280, splits=8),
    CV("conv_wgrad", 4, 28, 28, 512, 512, splits=0),
]

# VGG16 at batch 32: the classifier GEMMs (fwd with the automatic split, dX, dW) and the 3x3 layers that run on this kernel
VGG_FC = [(25088, 4096, True), (4096, 4096, True), (4096, 1000, False)]
VGG_CONV = [(64, 64, 224), (64, 128, 112), (128, 128, 112), (128, 256, 56), (256, 256, 56), (256, 512, 28), (512, 512, 28),
            (512, 512, 14)]


def _sms():
    """The SM count the library plans for: the device's, or 132 (its default) without one."""
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count if torch.cuda.is_available() else 132


def plan_of(c):
    """(instantiation key, plan, persistent) of a case, from the planners the launchers use."""
    op = c["op"]
    if op == "linear":
        s = tc_linear._auto_splits(c["M"], c["N"], c["K"], _sms()) if c["splits"] is None else c["splits"]
        p = tc_linear.plan(c["M"], c["N"], c["K"], reduce=s > 1, splits=s)
        entry = "linear_splitk" if s > 1 else "linear"
    elif op == "dgrad":
        p, entry = tc_linear.plan(c["M"], c["K"], c["N"]), "linear_dgrad"
    elif op == "wgrad":
        # (bnet_tc_plan wants the reduction padded to 8 like a K-major row pitch; the batch here is MN-major, any length works,
        #  and the tiling depends on its 64-row blocks only)
        p, entry = tc_linear.plan(c["N"], c["K"], -(-c["M"] // 8) * 8), "linear_wgrad"
    elif op in ("conv", "conv_dgrad"):
        p, entry = tc_conv.conv_plan(c["n"], c["h"], c["w"], c["cin"], c["cout"], dgrad=op == "conv_dgrad"), op
    else:
        p, entry = tc_conv.wgrad_plan(c["n"], c["h"], c["w"], c["cin"], c["cout"], c["splits"]), op
    tiles = p["grid_x"] * p["grid_y"]
    last_slice = p["k_blocks"] - (p["grid_z"] - 1) * p["k_per_split"]
    persistent = tiles >= 3 * p["ctas"] and (tiles // p["ctas"]) * last_slice > 2 * p["stages"]
    return (entry, p["bn"], p["swap"]), p, persistent


def vgg_cases():
    """The classifier GEMMs at batch 32, and one 3x3 case per distinct (instantiation, patch) that batch-32 VGG16 plans —
    at the smallest batch whose plan has the same instantiation, patch and persistence (the fp64 references stay cheap)."""
    cases = []
    for k, n, relu in VGG_FC:
        cases += [L("linear", 32, n, k, relu=relu, splits=None, name="vgg"), L("dgrad", 32, n, k, name="vgg"),
                  L("wgrad", 32, n, k, name="vgg")]
    seen = set()
    for cin, cout, hw in VGG_CONV:
        for op in ("conv", "conv_dgrad", "conv_wgrad"):
            def sig(b):
                key, p, pers = plan_of(CV(op, b, hw, hw, cin, cout))
                return key, (p.get("bw"), p.get("bh"), p.get("bn_images")) if op != "conv_wgrad" else (cin, cout, hw), pers
            want = sig(32)
            if want[:2] in seen:
                continue
            seen.add(want[:2])
            b = next(b for b in (1, 2, 4, 8, 16, 32) if sig(b) == want)
            cases.append(CV(op, b, hw, hw, cin, cout, relu=op == "conv", name=f"vgg{'' if b == 32 else f' (batch 32 as {b})'}"))
    return cases


def all_cases():
    return LINEAR_CASES + CONV_CASES + vgg_cases()


def describe(c):
    if "M" in c:
        s = f"{c['op']} M={c['M']} N={c['N']} K={c['K']}"
        s += f" splits={c['splits']}" if c["op"] == "linear" and c["splits"] != 1 else ""
    else:
        s = f"{c['op']} N={c['n']} {c['h']}x{c['w']} {c['cin']}->{c['cout']}" + (f" splits={c['splits']}" if c["op"] == "conv_wgrad" else "")
    s += " relu" if c.get("relu") and c["op"] in ("linear", "conv") else ""
    s += f" guarded(+{c['pad']})" if c["pad"] else ""
    return s + (f" [{c['name']}]" if c["name"] else "")


def job_coverage():
    """Every instantiation reached, every tile width persistent at least once — on the SMs of the device at hand, or 132
    (the host planner's default) without one."""
    print(f"planning for {_sms()} SMs")
    reached, persistent_bn = {}, set()
    for c in all_cases():
        key, _, pers = plan_of(c)
        reached.setdefault(key, []).append((describe(c), pers))
        if pers:
            persistent_bn.add(key[1])
    for key in sorted(reached):
        print(f"{key}: " + "; ".join(f"{d}{' (persistent)' if p else ''}" for d, p in reached[key]))
    missing = EXPECTED - set(reached)
    assert not missing, f"instantiations no case reaches: {sorted(missing)}"
    assert not set(reached) - EXPECTED, f"keys outside the dispatch tables: {sorted(set(reached) - EXPECTED)}"
    assert persistent_bn >= {32, 64, 128, 256}, f"tile widths never run persistent: {sorted({32, 64, 128, 256} - persistent_bn)}"
    print(json.dumps({"instantiations": len(reached), "persistent_bn": sorted(persistent_bn)}))


# ------------------------------------------------------------------------------------------------------------------- GPU side
SENT = 0x5A5A          # guard-band sentinel (int16 bits)
LEAD = 64              # guard elements before a flat output slice (128 bytes keeps the 16-byte alignment)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _int_operand(shape, red, g):
    """Sparse integers in {-2, -1, 1, 2}: about 48 nonzero products per output whatever the reduction length."""
    p = min(1.0, math.sqrt(48.0 / red))
    v = torch.randint(1, 3, shape, device="cuda", generator=g) * (torch.randint(0, 2, shape, device="cuda", generator=g) * 2 - 1)
    return (v * (torch.rand(shape, device="cuda", generator=g) < p)).to(torch.bfloat16)


def _operand(shape, red, g, exact, scale=1.0):
    if exact:
        return _int_operand(shape, red, g)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _bias(n, g, exact):
    if exact:
        return torch.randint(-4, 5, (n,), device="cuda", generator=g).to(torch.bfloat16)
    return torch.randn(n, device="cuda", generator=g).to(torch.bfloat16)


def _guarded(numel):
    """(flat int16 buffer filled with the sentinel, the bf16 slice of `numel` elements after LEAD guard elements)."""
    flat = torch.full((LEAD + numel + LEAD,), SENT, dtype=torch.int16, device="cuda")
    return flat, flat[LEAD:LEAD + numel]


def _check_guard(flat, region):
    """Everything of `flat` outside `region` (a view into it) still holds the sentinel."""
    chk = flat.clone()
    off = region.storage_offset() - flat.storage_offset()
    chk.as_strided(region.shape, region.stride(), chk.storage_offset() + off).fill_(SENT)
    bad = int((chk != SENT).sum().item())
    assert bad == 0, f"{bad} elements outside the output were written"


def _scratch_clean():
    for ws, cnt in list(tc_linear._scratch.values()) + list(tc_conv._wgrad_scratch.values()):
        assert not ws.any().item() and not cnt.any().item(), "split-K / fix-up scratch not handed back all zero"


def _run(c, ops):
    """One call of the kernel of case c on operands `ops`; returns (output as a bf16 tensor, guard check or None)."""
    op, pad = c["op"], c["pad"]
    if op == "linear":
        x, w, b = ops
        M, N = x.shape[0], w.shape[0]
        out = guard = None
        if pad:
            ld = N + pad
            flat, sl = _guarded(M * ld + ld)
            out = sl[ld:].view(M, ld)[:, :N].view(torch.bfloat16)
            guard = (flat, out.view(torch.int16))
        y = tc_linear.linear(x, w, b, c["relu"], out=out, splits=c["splits"])
        return y, guard
    if op == "dgrad":
        return tc_linear.linear_dgrad(*ops), None
    if op == "wgrad":
        gy, x = ops
        out = guard = None
        if pad:
            flat, sl = _guarded(gy.shape[1] * x.shape[1])
            out = sl.view(gy.shape[1], x.shape[1]).view(torch.bfloat16)
            guard = (flat, out.view(torch.int16))
        y = tc_linear.linear_wgrad(gy, x, out=out)
        assert out is None or y.data_ptr() == out.data_ptr(), "linear_wgrad did not write into out="
        return y, guard
    if op == "conv":
        x, w, b = ops
        n, _, h, wd = x.shape
        out = guard = None
        if pad:
            flat, sl = _guarded(n * h * wd * w.shape[0])
            out = sl.view(torch.bfloat16).view(n, h, wd, w.shape[0]).permute(0, 3, 1, 2)
            guard = (flat, sl)
        return tc_conv.conv3x3(x, w, b, relu=c["relu"], out=out), guard
    if op == "conv_dgrad":
        return tc_conv.conv3x3_dgrad(*ops), None
    gy, x = ops
    cout, cin = gy.shape[1], x.shape[1]
    out = guard = None
    if pad:
        flat, sl = _guarded(cout * 9 * cin)
        out = sl.view(torch.bfloat16).view(cout, 3, 3, cin).permute(0, 3, 1, 2)
        guard = (flat, sl)
    y = tc_conv.conv3x3_wgrad(gy, x, splits=c["splits"], out=out)
    assert out is None or y.data_ptr() == out.data_ptr(), "conv3x3_wgrad did not write into out="
    return y, guard


def _nhwc(t):
    return t.contiguous(memory_format=torch.channels_last)


def _operands(c, g, exact):
    """bf16 operands of case c, and the float64 reference of the op as a function of (operand transform, with bias)."""
    op = c["op"]
    if op in ("linear", "dgrad", "wgrad"):
        M, N, K = c["M"], c["N"], c["K"]
        if op == "linear":
            x, w = _operand((M, K), K, g, exact), _operand((N, K), K, g, exact, K ** -0.5)
            b = _bias(N, g, exact) if c["bias"] else None
            ops = (x, w, b)

            def ref(f, with_bias):
                r = f(x) @ f(w).t()
                return r + f(b) if (with_bias and b is not None) else r
        elif op == "dgrad":
            gy, w = _operand((M, N), N, g, exact), _operand((N, K), N, g, exact, N ** -0.5)
            ops = (gy, w)

            def ref(f, with_bias):
                return f(gy) @ f(w)
        else:
            gy, x = _operand((M, N), M, g, exact), _operand((M, K), M, g, exact, M ** -0.5)
            ops = (gy, x)

            def ref(f, with_bias):
                return f(gy).t() @ f(x)
        return ops, ref
    n, h, wd, cin, cout = c["n"], c["h"], c["w"], c["cin"], c["cout"]
    if op == "conv":
        x = _nhwc(_operand((n, cin, h, wd), 9 * cin, g, exact))
        w = _nhwc(_operand((cout, cin, 3, 3), 9 * cin, g, exact, (9 * cin) ** -0.5))
        b = _bias(cout, g, exact) if c["bias"] else None

        def ref(f, with_bias):
            return F.conv2d(f(x), f(w), f(b) if (with_bias and b is not None) else None, padding=1)
        return (x, w, b), ref
    if op == "conv_dgrad":
        gy = _nhwc(_operand((n, cout, h, wd), 9 * cout, g, exact))
        w = _nhwc(_operand((cout, cin, 3, 3), 9 * cout, g, exact, (9 * cout) ** -0.5))

        def ref(f, with_bias):
            return F.conv_transpose2d(f(gy), f(w), padding=1)
        return (gy, w), ref
    px = n * h * wd
    gy = _nhwc(_operand((n, cout, h, wd), px, g, exact))
    x = _nhwc(_operand((n, cin, h, wd), px, g, exact, px ** -0.5))

    def ref(f, with_bias):
        return torch.nn.grad.conv2d_weight(f(x), (cout, cin, 3, 3), f(gy), padding=1)
    return (gy, x), ref


def _f64(t):
    return None if t is None else t.double().contiguous()


def _abs64(t):
    return None if t is None else t.double().abs().contiguous()


def run_case(c, seed):
    """Exact and bounded checks of one case (plus guard bands and, for split reductions, three bit-identical calls).
    Returns (worst err / bound, persistent)."""
    key, p, pers = plan_of(c)
    repeat = 3 if key[0] in ("linear_splitk", "conv_wgrad") else 1
    relu = c.get("relu") and c["op"] in ("linear", "conv")
    worst = 0.0
    for exact in (True, False):
        g = _gen(seed * 2 + exact)
        ops, ref = _operands(c, g, exact)
        r = ref(_f64, True)
        if relu:
            r = torch.relu(r)
        outs = []
        for _ in range(repeat):
            y, guard = _run(c, ops)
            torch.cuda.synchronize()
            assert tc_linear.last_error() == 0, f"{describe(c)}: watchdog tripped"
            if guard is not None:
                _check_guard(*guard)
            _scratch_clean()
            outs.append(y.clone())
        for y2 in outs[1:]:
            assert torch.equal(y2.view(torch.int16), outs[0].view(torch.int16)), f"{describe(c)}: results differ between calls"
        y = outs[0]
        assert y.shape == r.shape, (y.shape, r.shape)
        if exact:
            amax = r.abs().max().item()
            assert amax <= 256, f"{describe(c)}: reference reaches {amax}, bf16 would not hold it exactly"
            want = r.to(torch.bfloat16)
            bad = (y != want)
            if bad.any():
                idx = bad.nonzero()[0].tolist()
                raise AssertionError(f"{describe(c)} key {key}: {int(bad.sum())} of {y.numel()} outputs differ from the exact result; "
                                     f"first at {idx}: got {y[tuple(idx)].item()} want {want[tuple(idx)].item()}")
        else:
            S = ref(_abs64, True)
            err = (y.double() - r).abs()
            bound = r.abs() * 2.0 ** -8 + S * 2.0 ** -16
            ratio = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))
            worst = ratio.max().item()
            assert worst <= 1.0, f"{describe(c)} key {key}: error reaches {worst:.3f} x the bound 2^-8 |r| + 2^-16 S"
        del ops, r
    return worst, pers


def _run_cases(cases, seed0):
    torch.cuda.set_device(0)
    assert tc_linear.supported(), "the wgmma kernels report unsupported on this GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    reached = {}
    for i, c in enumerate(cases):
        worst, pers = run_case(c, seed0 + i)
        key = plan_of(c)[0]
        print(f"{str(key):28s} {'persistent' if pers else 'one pass  '}  worst err/bound {worst:.3f}  {describe(c)}", flush=True)
        reached.setdefault(key, []).append(worst)
        torch.cuda.empty_cache()
    print(json.dumps({"keys": {str(k): max(v) for k, v in sorted(reached.items())}}), flush=True)


def job_linear():
    _run_cases(LINEAR_CASES, 100)


def job_conv():
    _run_cases(CONV_CASES, 200)


def job_vgg():
    _run_cases(vgg_cases(), 300)


# --------------------------------------------------------------------------------------------- NaN / Inf through the fused layers
def _same(a, b, what):
    """Equal values (+0 == -0), NaN in the same places."""
    assert a.shape == b.shape, (what, a.shape, b.shape)
    na, nb = a.isnan(), b.isnan()
    assert torch.equal(na, nb), f"{what}: NaN at {int((na != nb).sum())} different positions"
    assert torch.equal(a.masked_fill(na, 0), b.masked_fill(nb, 0)), f"{what}: {int((a.masked_fill(na, 0) != b.masked_fill(nb, 0)).sum())} values differ"


def _close(a, b, what, tol=6e-2):
    """NaN and +-Inf in the same places, the finite rest within a relative L2 error."""
    assert a.shape == b.shape, (what, a.shape, b.shape)
    a, b = a.float(), b.float()
    for name, fn in (("NaN", torch.isnan), ("+Inf", lambda t: t == math.inf), ("-Inf", lambda t: t == -math.inf)):
        assert torch.equal(fn(a), fn(b)), f"{what}: {name} at {int((fn(a) != fn(b)).sum())} different positions"
    fin = torch.isfinite(b)
    e = ((a[fin] - b[fin]).norm() / b[fin].norm().clamp_min(1e-6)).item()
    assert e < tol, f"{what}: relative L2 error {e}"


def _quarters(shape, g):
    """Multiples of 1/4 in [-2, 2]: z + b stays exact in bf16, so eager torch's rounding cannot create or break a tie."""
    return (torch.randint(-8, 9, shape, device="cuda", generator=g).float() / 4).to(torch.bfloat16)


def _sprinkle(t, g, frac=0.03):
    """NaN, +Inf and -Inf at random positions."""
    u = torch.rand(t.shape, device="cuda", generator=g)
    t = t.masked_fill(u < frac, float("nan"))
    t = t.masked_fill((u >= frac) & (u < 2 * frac), float("inf"))
    return t.masked_fill((u >= 2 * frac) & (u < 3 * frac), float("-inf"))


def job_nan():
    torch.cuda.set_device(0)
    g = _gen(11)
    lib, st = fused_nn._L(), fused_nn._stream()
    n, C, H, W = 3, 64, 6, 10
    # ---- bias + ReLU in place, isolated: bit-equal to eager (one rounding of z + b, then a monotone max)
    z = _nhwc(_sprinkle(_quarters((n, C, H, W), g), g))
    b = _quarters((C,), g)
    b[0], b[1], b[2] = float("nan"), float("inf"), float("-inf")
    y = z.clone()
    assert lib.bnet_nn_bias_relu(y.data_ptr(), b.data_ptr(), n * H * W, C, 1, st) == 1
    _same(y, torch.relu(z + b.view(1, C, 1, 1)), "bias_relu")
    # ---- bias + ReLU + 2x2 max-pool forward and backward, isolated; exact ties (first maximum wins) and windows holding two
    #      NaNs (torch routes the gradient to the last)
    z = _quarters((n, C, H, W), g)
    z[:, :, 0::2, 1::2] = z[:, :, 0::2, 0::2]                      # ties inside every window
    z[0, 3:9, 2, 4] = float("nan")
    z[0, 3:9, 3, 5] = float("nan")
    z = _nhwc(_sprinkle(z, g, 0.02))
    p = torch.empty((n, C, H // 2, W // 2), device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
    idx = torch.empty(p.numel(), device="cuda", dtype=torch.uint8)
    assert lib.bnet_nn_bias_relu_pool_fwd(z.data_ptr(), b.data_ptr(), p.data_ptr(), idx.data_ptr(), n, H, W, C, 1, st) == 1
    zr, br = z.clone().requires_grad_(), b.clone().requires_grad_()
    pr = F.max_pool2d(torch.relu(zr + br.view(1, C, 1, 1)), 2, 2)
    _same(p, pr.detach(), "bias_relu_pool forward")
    gp = _nhwc(_quarters(tuple(p.shape), g))
    pr.backward(gp)
    gz = torch.empty_like(z)
    gb = torch.zeros(C, device="cuda")
    assert lib.bnet_nn_pool_relu_bwd_bias_grad(gp.data_ptr(), idx.data_ptr(), gz.data_ptr(), gb.data_ptr(),
                                               fused_nn._partials(C, z.device).data_ptr(), n, H, W, C, 1, st) == 1
    _same(gz, zr.grad, "bias_relu_pool backward (input gradient)")
    _same(gb, gz.float().sum((0, 2, 3)), "bias_relu_pool backward (bias gradient = sum of the routed gradients)")
    # ---- ReLU backward: torch's threshold_backward (y <= 0 blocks, a NaN y passes), NaN gradients included
    yv = torch.relu(_nhwc(_sprinkle(_quarters((n, C, H, W), g), g, 0.05)))
    gy = _nhwc(_sprinkle(_quarters((n, C, H, W), g), g, 0.02))
    gz = torch.empty_like(gy)
    gb = torch.zeros(C, device="cuda")
    assert lib.bnet_nn_relu_bwd_bias_grad(gy.data_ptr(), yv.data_ptr(), gz.data_ptr(), gb.data_ptr(),
                                          fused_nn._partials(C, z.device).data_ptr(), n * H * W, C, 1, st) == 1
    want = torch.ops.aten.threshold_backward(gy, yv, 0)
    _same(gz, want, "relu backward")
    _same(gb, want.float().sum((0, 2, 3)), "relu backward (bias gradient)")
    print("fused bias/ReLU/pool kernels propagate NaN like eager torch", flush=True)

    # ---- the wgmma epilogue's ReLU: linear (and its autograd) and conv, NaN / +-Inf from the bias and a NaN activation
    x = torch.randn(48, 264, device="cuda", generator=g).bfloat16()
    x[5, 7] = float("nan")
    w = (torch.randn(136, 264, device="cuda", generator=g) / 16).bfloat16()
    b = torch.randn(136, device="cuda", generator=g).bfloat16()
    b[3], b[40], b[77] = float("nan"), float("inf"), float("-inf")
    xa, wa, ba = (t.clone().requires_grad_() for t in (x, w, b))
    ya = tc_linear.linear_bias_act(xa, wa, ba, True)
    assert tc_linear.last_error() == 0
    xb, wb, bb = (t.clone().requires_grad_() for t in (x, w, b))
    yb = torch.relu(F.linear(xb, wb, bb))
    _close(ya, yb, "linear + ReLU forward")
    go = torch.randn(ya.shape, device="cuda", generator=g).bfloat16()
    ya.backward(go)
    yb.backward(go)
    assert tc_linear.last_error() == 0
    for name, a_, b_ in (("dx", xa.grad, xb.grad), ("dw", wa.grad, wb.grad), ("db", ba.grad, bb.grad)):
        _close(a_, b_, f"linear + ReLU backward {name}")
    xc = torch.randn(2, 64, 9, 13, device="cuda", generator=g).bfloat16()
    xc[1, 5, 4, 6] = float("nan")
    xc = _nhwc(xc)
    wc = _nhwc((torch.randn(72, 64, 3, 3, device="cuda", generator=g) / 24).bfloat16())
    bc = torch.randn(72, device="cuda", generator=g).bfloat16()
    bc[0], bc[9], bc[33] = float("nan"), float("inf"), float("-inf")
    yc = tc_conv.conv3x3(xc, wc, bc, relu=True)
    assert tc_linear.last_error() == 0
    cols = F.unfold(xc.double(), 3, padding=1)                                     # plain dot products: IEEE NaN / Inf rules
    rc = (wc.double().reshape(72, -1) @ cols).view(2, 72, 9, 13) + bc.double().view(1, 72, 1, 1)
    _close(yc, torch.relu(rc), "conv3x3 + ReLU forward")
    print("wgmma epilogue ReLU propagates NaN like eager torch", flush=True)

    # ---- BatchNorm + residual + ReLU block: NaN / +-Inf arrive through the residual; forward values and autograd gradients
    import copy

    conv = torch.nn.Conv2d(64, 64, 3, 1, 1, bias=False).cuda().bfloat16().to(memory_format=torch.channels_last)
    bn_a = torch.nn.BatchNorm2d(64).cuda().bfloat16()
    bn_b = copy.deepcopy(bn_a)
    xs = _nhwc(torch.randn(4, 64, 8, 8, device="cuda", generator=g).bfloat16())
    res = _nhwc(_sprinkle(torch.randn(4, 64, 8, 8, device="cuda", generator=g).bfloat16(), g, 0.03))
    xa, ra = xs.clone().requires_grad_(), res.clone().requires_grad_()
    before = fused_nn.LAUNCHES
    ya = fused_nn.conv_bn_act(xa, conv, bn_a, relu=True, res=ra)
    assert fused_nn.LAUNCHES > before, "fused BatchNorm kernels did not run"
    go = _nhwc(torch.randn(ya.shape, device="cuda", generator=g).bfloat16())
    ya.backward(go)
    ga = [xa.grad.clone(), conv.weight.grad.clone(), bn_a.weight.grad.clone(), bn_a.bias.grad.clone(), ra.grad.clone()]
    conv.zero_grad(set_to_none=True)
    xb, rb = xs.clone().requires_grad_(), res.clone().requires_grad_()
    yb = torch.relu(bn_b(conv(xb)) + rb)
    yb.backward(go)
    gb_ = [xb.grad, conv.weight.grad, bn_b.weight.grad, bn_b.bias.grad, rb.grad]
    _close(ya, yb, "BN + residual + ReLU forward")
    for name, a_, b_ in zip(("dx", "dw", "dgamma", "dbeta", "dres"), ga, gb_):
        _close(a_, b_, f"BN + residual + ReLU backward {name}")
    print("fused BatchNorm + ReLU propagates NaN like eager torch", flush=True)


# --------------------------------------------------------------------------- ordered reductions of the fused layers: same bits
def job_reductions():
    """The bias-gradient and BatchNorm column reductions add per-block partial rows in block order: three calls on the same
    inputs give the same bits (the partial-row workspace is fresh, uninitialised memory every time)."""
    torch.cuda.set_device(0)
    g = _gen(23)
    lib, st = fused_nn._L(), fused_nn._stream()
    n, C, H, W = 16, 256, 56, 56
    rows = n * H * W
    gy = _nhwc(torch.randn(n, C, H, W, device="cuda", generator=g).bfloat16())
    y = torch.relu(_nhwc(torch.randn(n, C, H, W, device="cuda", generator=g).bfloat16()))
    gp = _nhwc(torch.randn(n, C, H // 2, W // 2, device="cuda", generator=g).bfloat16())
    idx = torch.randint(0, 8, (n * (H // 2) * (W // 2) * C,), device="cuda", generator=g).to(torch.uint8)

    def runs(fn):
        outs = [fn() for _ in range(3)]
        torch.cuda.synchronize()
        for o in outs[1:]:
            for a, b in zip(o, outs[0]):
                assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a.view(torch.int16),
                                   b.view(torch.int32) if b.dtype == torch.float32 else b.view(torch.int16)), "results differ between calls"
        return outs[0]

    def relu_bwd():
        gz, gb = torch.empty_like(gy), torch.zeros(C, device="cuda")
        assert lib.bnet_nn_relu_bwd_bias_grad(gy.data_ptr(), y.data_ptr(), gz.data_ptr(), gb.data_ptr(),
                                              fused_nn._partials(C, gy.device).data_ptr(), rows, C, 1, st) == 1
        return gz, gb

    def pool_bwd():
        gz, gb = torch.empty_like(gy), torch.zeros(C, device="cuda")
        assert lib.bnet_nn_pool_relu_bwd_bias_grad(gp.data_ptr(), idx.data_ptr(), gz.data_ptr(), gb.data_ptr(),
                                                   fused_nn._partials(C, gy.device).data_ptr(), n, H, W, C, 1, st) == 1
        return gz, gb

    def bn_stats():
        s = torch.zeros(2 * C, device="cuda")
        assert lib.bnet_nn_bn_stats(gy.data_ptr(), s.data_ptr(), fused_nn._partials(2 * C, gy.device).data_ptr(), rows, C, 1, st) == 1
        return (s,)

    stats = runs(bn_stats)[0]

    def bn_bwd():
        s = torch.zeros(2 * C, device="cuda")
        assert lib.bnet_nn_bn_bwd_reduce(gy.data_ptr(), y.data_ptr(), y.data_ptr(), stats.data_ptr(), s.data_ptr(),
                                         fused_nn._partials(2 * C, gy.device).data_ptr(), rows, C, 1e-5, 1, 1, st) == 1
        return (s,)

    gz, gb = runs(relu_bwd)
    want = gy.float().masked_fill(y <= 0, 0).sum((0, 2, 3))
    assert ((gb - want).abs() <= 1e-3 * want.abs().max()).all(), "relu backward bias gradient"
    gz, gb = runs(pool_bwd)
    routed = gp.float().permute(0, 2, 3, 1).reshape(-1, C).masked_fill((idx.view(-1, C) & 4) == 0, 0).sum(0)
    assert ((gb - routed).abs() <= 1e-3 * routed.abs().max()).all(), "pool backward bias gradient"
    # the statistics are sums of d = z - K and d^2, K = the channel's value in row 0; each sum within 1e-4 of its channel's sum of |terms|
    d = gy.double() - gy[0, :, 0, 0].double().view(1, C, 1, 1)
    ref = torch.cat([d.sum((0, 2, 3)), d.square().sum((0, 2, 3))])
    scale = torch.cat([d.abs().sum((0, 2, 3)), d.square().sum((0, 2, 3))])
    assert ((stats.double() - ref).abs() <= 1e-4 * scale).all(), "BatchNorm statistics (sums of z - K and (z - K)^2)"
    runs(bn_bwd)
    print("ordered column reductions: identical bits in 3 calls", flush=True)


JOBS = {k[4:]: v for k, v in globals().items() if k.startswith("job_")}

if __name__ == "__main__":
    JOBS[sys.argv[1]]()

"""Numerics of the fused layer kernels (csrc/cuda/nn_kernels.cu): bias + ReLU, 2x2 max-pool, their backward passes with the
bias-gradient reduction, and the four BatchNorm kernels, each called through its C entry point on tensors built here (no
convolution in the loop), against the same operation in float64 computed from the very values the kernel read.  Run by
tests/test_nn_numerics.py one job per child process: a kernel fault must not poison the pytest process, and the library reads
BNET_NN_BLOCKS_PER_SM (the reductions' grid cap) once per process.

Every output lives inside a larger buffer filled with a NaN sentinel: an element the kernel did not write still holds the
sentinel's bits, and a stray write before or after the output changes the guard.  The reductions' partial-row workspace is
filled with NaN too, so a partial row no block wrote turns the sum into NaN.

    python tests/nn_numerics_worker.py <job>          jobs: elementwise backward batchnorm nonfinite layer_gate
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bagua_net_b200.ops import fused_nn  # noqa: E402

DT = {torch.float32: 0, torch.bfloat16: 1}
VEC = {torch.float32: 4, torch.bfloat16: 8}
UNIT = {torch.float32: 2.0 ** -24, torch.bfloat16: 2.0 ** -8}   # unit roundoff of the output type
U32 = 2.0 ** -24
WIDTHS = (1, 3, 8, 17, 64, 100, 255, 256)                          # C / V: 16-byte channel vectors per pixel
LEAD = 64                                                          # guard elements on either side of an output
SENT = {torch.float32: (torch.int32, 0x7FA5A5A5), torch.bfloat16: (torch.int16, 0x7FA5), torch.uint8: (torch.uint8, 0xA5)}


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _cap():
    """Blocks of a reduce kernel at most: BNET_NN_BLOCKS_PER_SM (1..16, default 2) per SM, as nn_kernels.cu reads it."""
    try:
        v = int(os.environ.get("BNET_NN_BLOCKS_PER_SM", "2"))
    except ValueError:
        v = 2
    return min(max(v, 1), 16) * _sms()


def _reduce_grid(rows, cvec):
    """(grid, rows per block step, summation depth) of a column reduction, from the host's grid formula: at least 8 rows per
    thread per block, capped.  A column sum adds a thread's rows, the block's rpb threads, then ceil(grid / 8) partial rows in
    each of 8 lanes and the 8 lanes."""
    rpb = ((256 // cvec) * cvec) // cvec
    grid = max(1, min(-(-rows // (8 * rpb)), _cap()))
    depth = -(-rows // (grid * rpb)) + rpb + -(-grid // 8) + 8
    return grid, rpb, depth


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


class Guarded:
    """An output of `numel` elements inside a buffer filled with a NaN sentinel (LEAD elements on either side)."""

    def __init__(self, numel, dtype):
        self.dtype, self.numel = dtype, numel
        it, bits = SENT[dtype]
        self.flat = torch.full((LEAD + numel + LEAD,), bits, dtype=it, device="cuda")
        self.out = self.flat[LEAD:LEAD + numel].view(dtype)

    def nhwc(self, n, c, h, w):
        return self.out.view(n, h, w, c).permute(0, 3, 1, 2)

    def check(self, what):
        it, bits = SENT[self.dtype]
        g = torch.cat([self.flat[:LEAD], self.flat[LEAD + self.numel:]])
        assert bool((g == bits).all()), f"{what}: {int((g != bits).sum())} elements outside the output were written"
        inner = self.flat[LEAD:LEAD + self.numel]
        left = int((inner == bits).sum())
        assert left == 0, f"{what}: {left} of {self.numel} output elements were never written"


def _nhwc(t):
    return t.contiguous(memory_format=torch.channels_last)


def _partials(ld):
    return fused_nn._partials(ld, torch.device("cuda")).fill_(float("nan"))


def _rows_cases(cvec, grid_wrap=True):
    """1, rpb - 1, rpb, ragged tails of the 4-row batches, and (grid_wrap) more than 8 rpb cap rows: the grid is capped and every
    thread wraps, its last batch ragged."""
    rpb = ((256 // cvec) * cvec) // cvec
    rows = {1, max(1, rpb - 1), rpb, 3 * rpb * 4 + 1, 5 * rpb * 4 + rpb // 2 + 3}
    if grid_wrap:
        rows.add(8 * rpb * _cap() + 3 * rpb + 1)
    return sorted(rows)


def _eq(a, b, what):
    """Equal values (+0 == -0); NaN nowhere."""
    bad = a != b
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {a.numel()} differ; first at {i}: got {a[tuple(i)].item()} "
                             f"want {b[tuple(i)].item()}")


def _ratio(err, bound, what):
    """worst err / bound; fails above 1."""
    r = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))
    assert not bool(torch.isnan(r).any()), f"{what}: NaN in the error"
    worst = r.max().item()
    if worst > 1.0:
        i = (r == r.max()).nonzero()[0].tolist()
        raise AssertionError(f"{what}: error reaches {worst:.3f} x its bound (at {i}: err {err[tuple(i)].item():.4g}, "
                             f"bound {bound[tuple(i)].item():.4g})")
    return worst


# ------------------------------------------------------------------------------------------------------- bias + ReLU, pool forward
def _data(shape, g, dtype, exact, scale=1.0):
    """Small integers in [-4, 4] (exact sums, many ties) or Gaussian values, in dtype."""
    if exact:
        return torch.randint(-4, 5, shape, device="cuda", generator=g).to(dtype)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(dtype)


def check_bias_relu(n, h, w, cvec, dtype, g, exact):
    lib, st = fused_nn._L(), fused_nn._stream()
    C = cvec * VEC[dtype]
    z = _nhwc(_data((n, C, h, w), g, dtype, exact))
    b = _data((C,), g, dtype, exact, 0.5)
    buf = Guarded(z.numel(), dtype)
    y = buf.nhwc(n, C, h, w)
    y.copy_(z)
    assert lib.bnet_nn_bias_relu(y.data_ptr(), b.data_ptr(), n * h * w, C, DT[dtype], st) == 1
    torch.cuda.synchronize()
    buf.check("bias_relu")
    _eq(y, torch.relu(z.float() + b.float().view(1, C, 1, 1)).to(dtype), "bias_relu vs relu(z + b) rounded")


def check_pool_fwd(n, h, w, cvec, dtype, g, exact):
    lib, st = fused_nn._L(), fused_nn._stream()
    C = cvec * VEC[dtype]
    z = _nhwc(_data((n, C, h, w), g, dtype, exact))
    if exact:
        z[:, :, 0::2, 1::2] = z[:, :, 0::2, 0::2]               # more ties: the first maximum wins
    b = _data((C,), g, dtype, exact, 0.5)
    ho, wo = h // 2, w // 2
    pbuf, cbuf = Guarded(n * ho * wo * C, dtype), Guarded(n * ho * wo * C, torch.uint8)
    p = pbuf.nhwc(n, C, ho, wo)
    assert lib.bnet_nn_bias_relu_pool_fwd(z.data_ptr(), b.data_ptr(), p.data_ptr(), cbuf.out.data_ptr(), n, h, w, C,
                                          DT[dtype], st) == 1
    torch.cuda.synchronize()
    pbuf.check("pool forward values")
    cbuf.check("pool forward codes")
    code = cbuf.nhwc(n, C, ho, wo).long()
    u = z.float() + b.float().view(1, C, 1, 1)                  # what the kernel compares, in fp32
    a = torch.relu(u).to(dtype)
    _eq(p, F.max_pool2d(a.float(), 2, 2).to(dtype), "pool forward vs window max of rounded relu(z + b)")
    umax = F.max_pool2d(u, 2, 2)
    flows = ~(umax <= 0)
    _eq((code & 4) != 0, flows, "pool forward flow bit vs !(max <= 0)")
    pos = code & 3
    win = u.reshape(n, C, ho, 2, wo, 2).permute(0, 1, 2, 4, 3, 5).reshape(n, C, ho, wo, 4)
    picked = torch.gather(win, 4, pos.unsqueeze(-1)).squeeze(-1)
    _eq(picked, umax, "pool forward code points at the window's maximum")
    if exact:
        _, ti = F.max_pool2d(a.double().cpu(), 2, 2, return_indices=True)
        ti = ti.cuda()
        tpos = (ti // w - 2 * torch.arange(ho, device="cuda").view(1, 1, ho, 1)) * 2 + (ti % w - 2 * torch.arange(wo, device="cuda").view(1, 1, 1, wo))
        sel = umax > 0
        _eq(pos[sel], tpos[sel], "pool forward position vs max_pool2d(return_indices) where the max is > 0")


def job_elementwise():
    torch.cuda.set_device(0)
    g = _gen(1)
    wrap = 16 * _sms() * 256                                        # vectors of the elementwise kernels' largest grid
    for dtype in (torch.float32, torch.bfloat16):
        for cvec in WIDTHS:
            for exact in (True, False):
                # bias + ReLU: a few rows, ragged shapes, and more vectors than the grid has threads (the grid-stride loop wraps)
                for n, h, w in ((1, 1, 1), (3, 5, 7), (1, 1, -(-wrap * 5 // 4 // cvec))):
                    check_bias_relu(n, h, w, cvec, dtype, g, exact)
                # pool: H != W, H = W = 2, odd N, and one with more output vectors than grid threads
                big = -(-(wrap * 9 // 8) // (2 * cvec))            # output vectors: 2 rows of `big` pixels
                for n, h, w in ((1, 2, 2), (3, 4, 6), (5, 6, 2), (1, 4, 2 * big)):
                    check_pool_fwd(n, h, w, cvec, dtype, g, exact)
            print(f"{str(dtype):15s} C/V={cvec:3d}: bias_relu and pool forward exact (values, codes, guards)", flush=True)


# ---------------------------------------------------------------------------------------------- backward + bias-gradient reduction
def _gb_check(gb, routed, rows, cvec, exact, what):
    """gb (fp32, the library's sum) against the float64 sum of the routed gradients: exact on integer data, otherwise within
    2^-24 d sum|g| with d the summation depth."""
    ref = routed.double().sum(0)
    if exact:
        _eq(gb.double(), ref, f"{what} (exact on integers)")
        return 0.0
    _, _, depth = _reduce_grid(rows, cvec)
    return _ratio((gb.double() - ref).abs(), U32 * depth * routed.double().abs().sum(0), f"{what} bias gradient")


def check_relu_bwd(rows, cvec, dtype, g, exact):
    lib, st = fused_nn._L(), fused_nn._stream()
    C = cvec * VEC[dtype]
    gy = _data((rows, C), g, dtype, exact)
    y = torch.relu(_data((rows, C), g, dtype, exact))              # post-ReLU activations: many exact zeros
    gzb, gbb = Guarded(rows * C, dtype), Guarded(C, torch.float32)
    gb = gbb.out
    gb.zero_()
    assert lib.bnet_nn_relu_bwd_bias_grad(gy.data_ptr(), y.data_ptr(), gzb.out.data_ptr(), gb.data_ptr(), _partials(C).data_ptr(),
                                          rows, C, DT[dtype], st) == 1
    torch.cuda.synchronize()
    gzb.check("relu backward gz")
    gbb.check("relu backward gb")
    gz = gzb.out.view(rows, C)
    want = gy.masked_fill(y <= 0, 0)
    _eq(gz, want, "relu backward gz vs mask")
    return _gb_check(gb, want, rows, cvec, exact, "relu backward")


def check_pool_bwd(n, h, w, cvec, dtype, g, exact):
    lib, st = fused_nn._L(), fused_nn._stream()
    C = cvec * VEC[dtype]
    ho, wo = h // 2, w // 2
    gp = _data((n, ho, wo, C), g, dtype, exact)                  # NHWC storage order
    code = torch.randint(0, 8, (n, ho, wo, C), device="cuda", generator=g, dtype=torch.uint8)
    gzb, gbb = Guarded(n * h * w * C, dtype), Guarded(C, torch.float32)
    gb = gbb.out
    gb.zero_()
    assert lib.bnet_nn_pool_relu_bwd_bias_grad(gp.data_ptr(), code.data_ptr(), gzb.out.data_ptr(), gb.data_ptr(),
                                               _partials(C).data_ptr(), n, h, w, C, DT[dtype], st) == 1
    torch.cuda.synchronize()
    gzb.check("pool backward gz (every element of each 2x2 window)")
    gbb.check("pool backward gb")
    routed = gp.masked_fill((code & 4) == 0, 0)
    want = torch.zeros(n, ho, wo, 2, 2, C, device="cuda", dtype=dtype)
    q = (code & 3).long()
    for dy in range(2):
        for dx in range(2):
            want[:, :, :, dy, dx] = routed.masked_fill(q != dy * 2 + dx, 0)
    want = want.permute(0, 1, 3, 2, 4, 5).reshape(n, h, w, C)
    _eq(gzb.out.view(n, h, w, C), want, "pool backward gz vs scatter through the codes")
    return _gb_check(gb, routed.view(-1, C), n * ho * wo, cvec, exact, "pool backward")


def job_backward():
    torch.cuda.set_device(0)
    g = _gen(2)
    print(f"reduce grid cap {_cap()} blocks", flush=True)
    for dtype in (torch.float32, torch.bfloat16):
        for cvec in WIDTHS:
            worst = 0.0
            for exact in (True, False):
                for rows in _rows_cases(cvec):
                    worst = max(worst, check_relu_bwd(rows, cvec, dtype, g, exact))
                rpb = ((256 // cvec) * cvec) // cvec
                big = 8 * rpb * _cap() + rpb + 1                 # pooled rows: 1 x big, above 8 rpb cap
                for n, h, w in ((1, 2, 2), (3, 4, 6), (5, 6, 2), (1, 2, 2 * big)):
                    worst = max(worst, check_pool_bwd(n, h, w, cvec, dtype, g, exact))
            print(f"{str(dtype):15s} C/V={cvec:3d}: relu / pool backward gz exact, gb exact on integers; "
                  f"Gaussian gb worst err/bound {worst:.3f}", flush=True)


# ------------------------------------------------------------------------------------------------------------------- BatchNorm
RATIOS = (0.0, 16.0, 256.0, 1024.0)


def bn_data(rows, C, dtype, g):
    """z[rows, C] with channels far from zero.  fp32: channel c is off + sd N(0, 1) with off / sd cycling through RATIOS.
    bf16: Gaussian channels (off / sd 0 or 16) and channels of two or three adjacent bf16 values around 2^e (mean / std near
    2^7 - 2^8).  The last channel (of more than one) is constant."""
    c = torch.arange(C, device="cuda")
    sd = torch.pow(2.0, (c % 7 - 3).double())
    e = torch.randn(rows, C, device="cuda", generator=g, dtype=torch.float64)
    if dtype == torch.float32:
        z = torch.tensor(RATIOS, device="cuda", dtype=torch.float64)[c % 4] * sd + sd * e
    else:
        kind = c % 4
        z = torch.where(kind == 1, 16 * sd, 0 * sd) + sd * e
        j = torch.randint(0, 3, (rows, C), device="cuda", generator=g).double()
        j = torch.where(kind == 2, j.clamp(max=1), j)
        adj = torch.pow(2.0, (c % 9 - 4).double()) * (1 + j / 128)
        z = torch.where(kind >= 2, adj, z)
    if C > 1:
        z[:, -1] = 3.0 * sd[-1]
    return z.to(dtype)


def check_batchnorm(rows, cvec, dtype, g, relu, with_res):
    lib, st = fused_nn._L(), fused_nn._stream()
    V = VEC[dtype]
    C = cvec * V
    uo = UNIT[dtype]
    eps = 1e-5
    z = bn_data(rows, C, dtype, g)
    gamma = ((torch.rand(C, device="cuda", generator=g) + 0.5) * torch.where(torch.rand(C, device="cuda", generator=g) < 0.2, -1, 1)).to(dtype)
    beta = (torch.randn(C, device="cuda", generator=g) * 0.5).to(dtype)
    res = torch.randn(rows, C, device="cuda", generator=g).to(dtype) if with_res else None
    gy = torch.randn(rows, C, device="cuda", generator=g).to(dtype)
    grid, rpb, depth = _reduce_grid(rows, cvec)

    # ---- statistics
    stats = torch.zeros(2 * C, device="cuda")
    assert lib.bnet_nn_bn_stats(z.data_ptr(), stats.data_ptr(), _partials(2 * C).data_ptr(), rows, C, DT[dtype], st) == 1
    z64 = z.double()
    worst = {}

    # ---- apply, momentum 1: running_mean = the kernel's mean, running_var = its variance * rows / (rows - 1)
    m = z64[0] + (z64 - z64[0]).mean(0)             # (exact on a constant channel, where v is then exactly 0)
    v = (z64 - m).square().mean(0)
    sd = v.sqrt()
    const = v == 0
    dm = torch.where(const, torch.zeros_like(m), 2.0 ** -22 * m.abs() + 2.0 ** -20 * sd)   # the statistics' contract
    dv = 2.0 ** -16 * v
    rm = torch.full((C,), 7.0, device="cuda", dtype=dtype)
    rv = torch.full((C,), 7.0, device="cuda", dtype=dtype)
    yb = Guarded(rows * C, dtype)
    assert lib.bnet_nn_bn_apply(z.data_ptr(), res.data_ptr() if with_res else None, yb.out.data_ptr(), stats.data_ptr(),
                                gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr(), rows, C, eps, 1.0,
                                int(relu), DT[dtype], st) == 1
    torch.cuda.synchronize()
    yb.check("bn_apply y")
    unb = rows / (rows - 1) if rows > 1 else 1.0
    rm64, rv64 = rm.double(), rv.double()
    worst["mean"] = _ratio((rm64 - m).abs(), dm + uo * (m.abs() + dm), "mean (running_mean, momentum 1)")
    verr, vbound = (rv64 - v * unb).abs(), unb * dv + (uo + 3 * U32) * v * unb
    over = verr > vbound
    if bool(over.any()):
        offs = sorted({f"{x:.0f}" for x in (m.abs() / sd.clamp_min(1e-300))[over].tolist()}, key=float)
        raise AssertionError(f"variance (running_var / unbias, momentum 1): error above 2^-16 var in {int(over.sum())} of {C} channels, "
                             f"at mean/std {offs}; worst {(verr / vbound)[over].max().item():.3g} x the bound")
    worst["var"] = _ratio(verr, vbound, "variance")
    assert bool((rv64[const] == 0).all()), "a constant channel's variance is not 0"
    # the statistics buffer: sums of d = z - K, K = row 0 of the channel
    d = z64 - z64[0]
    worst["stats"] = max(_ratio((stats[:C].double() - d.sum(0)).abs(), U32 * (depth + 1) * d.abs().sum(0), "bn_stats sum of z - K"),
                         _ratio((stats[C:].double() - d.square().sum(0)).abs(), U32 * (depth + 2) * d.square().sum(0),
                                "bn_stats sum of (z - K)^2"))
    y = yb.out.view(rows, C)
    inv = 1.0 / (v + eps).sqrt()
    di = dv / (2 * (v + eps)) + 6 * U32          # relative error of the kernel's invstd (rsqrtf: 2 ulp, v + eps: 1/2 ulp)
    g64, b64 = gamma.double(), beta.double()
    xh = (z64 - m) * inv
    ex = inv * dm + xh.abs() * (di + 4 * U32)                               # error of the kernel's xhat
    t = g64 * xh + b64 + (res.double() if with_res else 0)
    r = torch.relu(t) if relu else t
    bt = g64.abs() * ex + 4 * U32 * ((g64 * xh).abs() + b64.abs() + (res.double().abs() if with_res else 0) + t.abs())
    worst["y"] = _ratio((y.double() - r).abs(), bt * (1 + uo) + uo * r.abs(), "bn_apply y")
    if bool(const.any()):
        cy = (b64 + (res.double() if with_res else torch.zeros_like(z64)))[:, const]
        cy = torch.relu(cy) if relu else cy
        _ratio((y.double()[:, const] - cy).abs(), 4 * U32 * cy.abs() * (1 + uo) + uo * cy.abs(), "bn_apply y of a constant channel vs beta")

    # ---- backward reduce and apply, on the kernel's y
    gsum = torch.zeros(2 * C, device="cuda")
    assert lib.bnet_nn_bn_bwd_reduce(gy.data_ptr(), y.data_ptr(), z.data_ptr(), stats.data_ptr(), gsum.data_ptr(),
                                     _partials(2 * C).data_ptr(), rows, C, eps, int(relu), DT[dtype], st) == 1
    gzb = Guarded(rows * C, dtype)
    grb = Guarded(rows * C, dtype) if with_res else None
    dgb, dbb = Guarded(C, dtype), Guarded(C, dtype)
    assert lib.bnet_nn_bn_bwd_apply(gy.data_ptr(), y.data_ptr(), z.data_ptr(), gzb.out.data_ptr(),
                                    grb.out.data_ptr() if with_res else None, stats.data_ptr(), gsum.data_ptr(), gamma.data_ptr(),
                                    dgb.out.data_ptr(), dbb.out.data_ptr(), rows, C, eps, int(relu), DT[dtype], st) == 1
    torch.cuda.synchronize()
    for buf, what in ((gzb, "gz"), (dgb, "dgamma"), (dbb, "dbeta")) + (((grb, "gres"),) if with_res else ()):
        buf.check(f"bn backward {what}")
    dy = gy.masked_fill(y <= 0, 0) if relu else gy
    if with_res:
        _eq(grb.out.view(rows, C), dy, "bn backward gres vs the masked gradient")
    dy64 = dy.double()
    r1, r2 = dy64.sum(0), (dy64 * xh).sum(0)
    b1 = U32 * depth * dy64.abs().sum(0)
    b2 = (dy64.abs() * ex).sum(0) + U32 * (depth + 2) * (dy64 * xh).abs().sum(0)
    worst["dbeta"] = _ratio((gsum[:C].double() - r1).abs(), b1, "bn backward s1 = dbeta")
    worst["dgamma"] = _ratio((gsum[C:].double() - r2).abs(), b2, "bn backward s2 = dgamma")
    _eq(dbb.out, gsum[:C].to(dtype), "dbeta vs s1 rounded")
    _eq(dgb.out, gsum[C:].to(dtype), "dgamma vs s2 rounded")
    c1, c2 = r1 / rows, r2 / rows
    dc1, dc2 = b1 / rows + 2 * U32 * c1.abs(), b2 / rows + 2 * U32 * c2.abs()
    inner = dy64 - c1 - xh * c2
    dinner = dc1 + xh.abs() * dc2 + ex * c2.abs() + 4 * U32 * (dy64.abs() + c1.abs() + (xh * c2).abs())
    a = g64 * inv
    gz64 = a * inner
    bg = a.abs() * dinner + a.abs() * (di + U32) * inner.abs()
    worst["gz"] = _ratio((gzb.out.view(rows, C).double() - gz64).abs(), bg * (1 + uo) + uo * gz64.abs(), "bn backward gz")
    return worst


def job_batchnorm():
    torch.cuda.set_device(0)
    g = _gen(3)
    print(f"reduce grid cap {_cap()} blocks", flush=True)
    combos = ((True, False), (False, False), (True, True), (False, True))
    for dtype in (torch.float32, torch.bfloat16):
        for cvec in WIDTHS:
            rpb = ((256 // cvec) * cvec) // cvec
            rows_list = sorted({2, max(2, rpb - 1), 3 * rpb * 4 + 1, 5 * rpb * 4 + rpb // 2 + 3, 8 * rpb * _cap() + 3 * rpb + 1})
            worst = {}
            for i, rows in enumerate(rows_list):
                for relu, with_res in (combos if rows <= 4 * rpb * 4 else combos[i % 4:i % 4 + 1]):
                    for k, x in check_batchnorm(rows, cvec, dtype, g, relu, with_res).items():
                        worst[k] = max(worst.get(k, 0.0), x)
            print(f"{str(dtype):15s} C/V={cvec:3d} rows {rows_list}: worst err/bound " +
                  " ".join(f"{k} {x:.3f}" for k, x in worst.items()), flush=True)


# ---------------------------------------------------------------------------------------------------- non-finite values in z
def job_nonfinite():
    """NaN or +-Inf in one channel of z, in row 0 (the statistics' pivot) or further down: y and running_var have NaN where
    eager BatchNorm2d (+ residual + ReLU) has them."""
    torch.cuda.set_device(0)
    lib, st = fused_nn._L(), fused_nn._stream()
    g = _gen(4)
    for dtype in (torch.float32, torch.bfloat16):
        n, h, w = 2, 5, 7
        C = 8 * VEC[dtype]
        for relu, with_res in ((True, True), (False, False)):
            z = torch.randn(n, C, h, w, device="cuda", generator=g).to(dtype)
            z[0, 1, 0, 0] = float("nan")                 # pivot
            z[1, 2, 3, 4] = float("inf")
            z[0, 3, 0, 0] = float("-inf")                # pivot
            z[0, 4, 0, 0] = float("inf")                 # pivot
            z[1, 5, 2, 1] = float("nan")
            z[1, 6, 1, 1] = float("-inf")
            z[0, 7, 2, 2], z[1, 7, 4, 6] = float("inf"), float("-inf")
            z = _nhwc(z)
            res = _nhwc(torch.randn(n, C, h, w, device="cuda", generator=g).to(dtype)) if with_res else None
            gamma = (torch.rand(C, device="cuda", generator=g) + 0.5).to(dtype)
            beta = torch.randn(C, device="cuda", generator=g).to(dtype)
            rows = n * h * w
            stats = torch.zeros(2 * C, device="cuda")
            assert lib.bnet_nn_bn_stats(z.data_ptr(), stats.data_ptr(), _partials(2 * C).data_ptr(), rows, C, DT[dtype], st) == 1
            rm, rv = torch.zeros(C, device="cuda", dtype=dtype), torch.ones(C, device="cuda", dtype=dtype)
            y = torch.empty_like(z)
            assert lib.bnet_nn_bn_apply(z.data_ptr(), res.data_ptr() if with_res else None, y.data_ptr(), stats.data_ptr(),
                                        gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(), rv.data_ptr(), rows, C, 1e-5, 0.1,
                                        int(relu), DT[dtype], st) == 1
            erm, erv = torch.zeros(C, device="cuda", dtype=dtype), torch.ones(C, device="cuda", dtype=dtype)
            ey = F.batch_norm(z, erm, erv, gamma, beta, training=True, momentum=0.1, eps=1e-5)
            if with_res:
                ey = ey + res
            if relu:
                ey = torch.relu(ey)
            torch.cuda.synchronize()
            for what, a, b in (("y", y, ey), ("running_var", rv, erv)):
                na, nb = a.isnan(), b.isnan()
                assert torch.equal(na, nb), (f"{dtype} relu={relu} res={with_res}: {what} NaN at {int((na != nb).sum())} positions "
                                             f"other than eager torch's (channels {sorted(set((na != nb).nonzero()[:, 1 if a.dim() > 1 else 0].tolist()))})")
            assert bool(rv[8:].isfinite().all()), "finite channels got a non-finite running_var"
            print(f"{str(dtype):15s} relu={relu} res={with_res}: NaN pattern of y and running_var as in eager torch", flush=True)


# ------------------------------------------------------------------------------------------------------- channel-width gate
def job_layer_gate():
    """ConvBiasReLU with 257 16-byte channel vectors (wider than the reduce kernels take) falls back to eager and matches it,
    forward and backward; at 256 it takes the fused path."""
    torch.cuda.set_device(0)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g = _gen(5)
    for dtype in (torch.float32, torch.bfloat16):
        V = VEC[dtype]
        for cvec in (256, 257):
            for pool in (False, True):
                torch.manual_seed(7)
                blk = fused_nn.ConvBiasReLU(16, cvec * V, 1, 1, 0, pool=pool).cuda().to(dtype).to(memory_format=torch.channels_last)
                x = _nhwc(torch.randn(2, 16, 4, 6, device="cuda", generator=g).to(dtype))
                xa, xb = x.clone().requires_grad_(), x.clone().requires_grad_()
                before = fused_nn.LAUNCHES
                ya = blk(xa)
                go = torch.randn(ya.shape, device="cuda", generator=g).to(dtype)
                ya.backward(go)
                fused = fused_nn.LAUNCHES > before
                ga = [xa.grad.float(), blk.conv.weight.grad.float().clone(), blk.conv.bias.grad.float().clone()]
                blk.zero_grad(set_to_none=True)
                yb = torch.relu(blk.conv(xb))
                if pool:
                    yb = F.max_pool2d(yb, 2, 2)
                yb.backward(go)
                gb = [xb.grad.float(), blk.conv.weight.grad.float(), blk.conv.bias.grad.float()]
                torch.cuda.synchronize()
                assert fused == (cvec <= 256), f"{dtype} C/V={cvec} pool={pool}: fused path taken: {fused}"
                # (bf16: the fused pool compares z + b before rounding, eager after, so near-ties route a few gradients differently)
                tol = 1e-5 if dtype == torch.float32 else 6e-2
                for name, a_, b_ in (("y", ya.float(), yb.float()), ("dx", ga[0], gb[0]), ("dw", ga[1], gb[1]), ("db", ga[2], gb[2])):
                    e = ((a_ - b_).norm() / b_.norm().clamp_min(1e-12)).item()
                    assert e < tol, f"{dtype} C/V={cvec} pool={pool}: {name} relative L2 error {e}"
                print(f"{str(dtype):15s} C/V={cvec} pool={pool}: {'fused' if fused else 'eager'}, matches eager torch", flush=True)


JOBS = {k[4:]: v for k, v in globals().items() if k.startswith("job_")}

if __name__ == "__main__":
    JOBS[sys.argv[1]]()

"""Per-rank bodies of the all-reduce numerics tests (launched by tests/test_allreduce_numerics.py, one process per GPU).

Every kernel result is compared element by element with a float64 reduction of the inputs as the kernel sees them
(rounded to the dtype), within the bound its fp32 arithmetic allows:

    sum:  gamma_{W-1} A (1 + u_dt) + u_dt |S| + F
    avg:  (gamma_{W-1} A + F) m / W + (m - 1) |S| / W + F,   m = (1 + u32)^2 (1 + u_dt)^k
    max, min: exact

S is the float64 sum over the ranks, A the sum of the absolute values, u32 = 2^-24, u_dt the dtype's unit roundoff,
F the dtype's smallest subnormal, gamma_n = n u32 / (1 - n u32).  k = 1 for the peer-load, one-shot and LL kernels
(the fp32 sum times fl(1/W) rounded once to the dtype) and k = 2 for the in-switch kernel, whose switch returns the sum
rounded to the dtype before the kernel scales it.  The in-switch sum is assumed to accumulate in fp32 and round once
(`.acc::f32`)."""
from __future__ import annotations

import ctypes as C
import math
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

QUICK = os.environ.get("BNET_TEST_QUICK") == "1"      # under compute-sanitizer: same code paths, smaller tensors
RANK = int(os.environ.get("RANK", "0"))
WORLD = int(os.environ.get("WORLD_SIZE", "1"))
LOCAL = int(os.environ.get("LOCAL_RANK", "0"))

DTYPES = (torch.float32, torch.bfloat16, torch.float16)
OPS = ("sum", "avg", "max", "min")
U32 = 2.0 ** -24
UDT = {torch.float32: 2.0 ** -24, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
FMIN = {torch.float32: 2.0 ** -149, torch.bfloat16: 2.0 ** -133, torch.float16: 2.0 ** -24}
EXP = {torch.float32: 20, torch.bfloat16: 20, torch.float16: 9}     # inputs are N(0, 1) * 2^k, |k| <= EXP (f16: no overflow)
GUARD = 256                                                          # guard bytes before every tensor (16-byte aligned)
SENTINEL = (0x5B + 16 * RANK) & 0xFF                                 # rank-specific guard byte
HEAP = 256 << 20                                                     # enough for every job at eight ranks
GRIDS = (1, 0) if QUICK else (1, 7, 132, 0)                          # 0: the communicator's default grid


def setup():
    torch.cuda.set_device(LOCAL)
    dist.init_process_group("nccl")                 # also at one rank: the jobs compare with NCCL's results


def teardown():
    dist.barrier()
    dist.destroy_process_group()


def sync():
    torch.cuda.synchronize()
    dist.barrier()


def bits(t):
    return t.contiguous().view(torch.uint8)


def same_on_every_rank(t: torch.Tensor) -> bool:
    if WORLD == 1:
        return True
    lst = [torch.empty_like(bits(t)) for _ in range(WORLD)]
    dist.all_gather(lst, bits(t))
    return all(torch.equal(lst[0], x) for x in lst)


# ------------------------------------------------------------------ inputs and the float64 reference
def rank_inputs(seed, n, dtype):
    """Every rank's input of one call, rounded to `dtype`: N(0, 1) * 2^k with k per element in [-EXP, EXP] (the exponents
    spread, so sums cancel: A >> |S|), exact +-pairs across ranks (rank r and rank W-1-r), zeros on even ranks, and
    subnormals of the dtype."""
    i = torch.arange(n, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(seed)
    shared = torch.randn(n, device="cuda", generator=g, dtype=torch.float64)
    shared = (shared * torch.exp2(torch.randint(-EXP[dtype], EXP[dtype] + 1, (n,), device="cuda", generator=g).double())).to(dtype)
    xs = []
    for r in range(WORLD):
        g = torch.Generator(device="cuda").manual_seed(seed * 64 + r + 1)
        x = torch.randn(n, device="cuda", generator=g, dtype=torch.float64)
        x = x * torch.exp2(torch.randint(-EXP[dtype], EXP[dtype] + 1, (n,), device="cuda", generator=g).double())
        sub = torch.randint(-64, 65, (n,), device="cuda", generator=g).double() * FMIN[dtype]
        x = torch.where(i % 11 == 3, sub, x).to(dtype)
        pair = shared if r < WORLD - 1 - r else (-shared if r > WORLD - 1 - r else torch.zeros_like(shared))
        x = torch.where(i % 5 == 1, pair, x)
        if r % 2 == 0:
            x = torch.where(i % 7 == 2, torch.zeros_like(x), x)
        xs.append(x)
    return xs


def bound(X, op, dtype, k):
    """The element-wise bound of the module docstring for the float64 stack X of every rank's inputs; k = 1 or 2."""
    S, A = X.sum(0), X.abs().sum(0)
    udt, F = UDT[dtype], FMIN[dtype]
    gamma = (WORLD - 1) * U32 / (1 - (WORLD - 1) * U32)
    if op == "sum":
        return S, gamma * A * (1 + udt) + udt * S.abs() + F
    m = (1 + U32) ** 2 * (1 + udt) ** k
    return S / WORLD, (gamma * A + F) * m / WORLD + (m - 1) * S.abs() / WORLD + F


class Checker:
    """Compares results with the float64 reference and keeps the worst error/bound per (W, path, dtype, op)."""

    def __init__(self):
        self.worst = {}

    def check(self, got, xs, op, dtype, path, what):
        X = torch.stack([x.double() for x in xs])
        key = (WORLD, path, str(dtype).split(".")[-1], op)
        if op in ("max", "min"):
            want = X.max(0).values if op == "max" else X.min(0).values
            bad = int((got.double() != want).sum())
            assert bad == 0, f"{what}: {bad} elements differ from the exact {op}"
            self.worst[key] = max(self.worst.get(key, 0.0), 0.0)
            return
        want, b = bound(X, op, dtype, 2 if path == "nvls" else 1)
        r = ((got.double() - want).abs() / b).nan_to_num(nan=math.inf, posinf=math.inf)
        w = float(r.max()) if r.numel() else 0.0
        self.worst[key] = max(self.worst.get(key, 0.0), w)
        if w > 1.0:
            j = int(r.argmax())
            raise AssertionError(f"{what}: error/bound {w:.3f} at element {j}: got {float(got[j])!r}, float64 "
                                 f"{float(want[j])!r}, bound {float(b[j]):.3e}, inputs {X[:, j].tolist()}")

    def report(self, job):
        if RANK == 0:
            for (w, path, dt, op), v in sorted(self.worst.items()):
                print(f"{job}: W={w} {path:8s} {dt:9s} {op:4s} worst error/bound {v:.4f}", flush=True)


class Arena:
    """A byte buffer (in the symmetric heap or ordinary device memory) whose bytes outside the tensor placed in it hold
    the rank's sentinel: a store at a wrong offset, by this rank or a peer, shows in `check`."""

    def __init__(self, comm, nbytes, heap):
        n = GUARD + nbytes + GUARD
        self.buf = comm.alloc(n, torch.uint8) if heap else torch.empty(n, dtype=torch.uint8, device="cuda")
        self.used = 0

    def window(self, n, dtype):
        """Fill with the sentinel and return the tensor of n elements after the leading guard (sentinel bytes too, so an
        element a kernel fails to write shows as wrong)."""
        self.buf.fill_(SENTINEL)
        self.lo, self.used = GUARD, n * torch.empty((), dtype=dtype).element_size()
        return self.buf[GUARD:GUARD + self.used].view(dtype)

    def place(self, x):
        """`window` holding a copy of x."""
        v = self.window(x.numel(), x.dtype)
        v.copy_(x)
        return v

    def check(self, what):
        lo, hi = self.lo, self.lo + self.used
        ok = bool((self.buf[:lo] == SENTINEL).all()) and bool((self.buf[hi:] == SENTINEL).all())
        assert ok, f"{what}: a guard byte around the tensor was overwritten on rank {RANK}"


def unroll(path):
    """Vectors per thread per round of the body that runs at this world size."""
    if path == "nvls":
        return 8
    return {2: 4, 4: 4, 8: 2}.get(WORLD, 1)


def per_rank_sizes(path):
    """16-byte vectors per rank: tiny, one short of / exactly / one past a full round of 1 and 7 CTAs, and one size that
    reaches the default grid of 132 CTAs (and the in-switch default of 32)."""
    u = unroll(path)
    s = {1, 2, 5}
    for nb in (1, 7):
        s |= {u * nb * 512 - 1, u * nb * 512, u * nb * 512 + 1}
    if not QUICK:
        s.add(132 * 1024 + 5)
    return sorted(s)


def elems(dtype):
    return 16 // torch.empty((), dtype=dtype).element_size()


# ------------------------------------------------------------------ jobs
def job_probe():
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(64 << 20)
    print(f"rank {RANK}: multicast={comm.has_multicast}", flush=True)
    teardown()


def job_twoshot():
    """The in-place heap all-reduces: two-shot peer loads/stores, and the in-switch kernel when there is multicast."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(HEAP)
    paths = ["p2p"] + (["nvls"] if comm.has_multicast else [])
    arena = Arena(comm, 16 * WORLD * max(max(per_rank_sizes(p)) for p in paths), heap=True)
    chk = Checker()
    nvls_repeat = {}
    seed = 0
    for path in paths:
        for dtype in DTYPES:
            for per in per_rank_sizes(path):
                n = per * WORLD * elems(dtype)
                seed += 1
                xs = rank_inputs(seed, n, dtype)
                for op in OPS:
                    first = None
                    for nb in GRIDS + ((0,) if path == "nvls" else ()):
                        t = arena.place(xs[RANK])
                        sync()
                        comm.all_reduce(t, op, algo=path, nblocks=nb)
                        torch.cuda.synchronize()
                        what = f"{path} {dtype} {op} {per} vectors/rank nblocks={nb}"
                        arena.check(what)
                        chk.check(t, xs, op, dtype, path, what)
                        assert same_on_every_rank(t), f"{what}: ranks hold different bits"
                        if first is None:
                            first = t.clone()
                        elif path == "nvls" and op in ("sum", "avg"):
                            nvls_repeat[(dtype, op)] = nvls_repeat.get((dtype, op), True) and torch.equal(bits(first), bits(t))
                        else:
                            assert torch.equal(bits(first), bits(t)), f"{what}: bits differ from nblocks={GRIDS[0]}"
    assert comm.status() == 0
    chk.report("twoshot")
    if RANK == 0:
        print(f"twoshot: W={WORLD} multicast={comm.has_multicast}; in-switch repeats gave the same bits: "
              f"{ {str(k[0]).split('.')[-1] + ' ' + k[1]: v for k, v in nvls_repeat.items()} or 'not run'}", flush=True)
    teardown()


def job_oneshot():
    """The one-shot kernel (every rank reads every peer, out of place): inputs unchanged, `out` guarded, sizes that are
    not a multiple of the world size, and both rejections of bad arguments (no launch)."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(HEAP)
    sizes = sorted({v * WORLD for v in per_rank_sizes("p2p")} | {1, 3, 7 * 512 + 3, 512 * WORLD + 1})
    src = Arena(comm, 16 * max(sizes), heap=True)
    dst = Arena(comm, 16 * max(sizes), heap=False)
    chk = Checker()
    seed = 1000
    for dtype in DTYPES:
        for nvec in sizes:
            n = nvec * elems(dtype)
            seed += 1
            xs = rank_inputs(seed, n, dtype)
            for op in OPS:
                first = None
                for nb in GRIDS:
                    t = src.place(xs[RANK])
                    out = dst.window(n, dtype)
                    sync()
                    comm.all_reduce_oneshot(t, out, op, nblocks=nb)
                    sync()                              # (no rank refills its input before every peer has read it)
                    what = f"oneshot {dtype} {op} {nvec} vectors nblocks={nb}"
                    src.check(what + " (input)")
                    dst.check(what + " (out)")
                    assert torch.equal(bits(t), bits(xs[RANK])), f"{what}: the heap input changed"
                    chk.check(out, xs, op, dtype, "oneshot", what)
                    assert same_on_every_rank(out), f"{what}: ranks hold different bits"
                    if first is None:
                        first = out.clone()
                    assert torch.equal(bits(first), bits(out)), f"{what}: bits differ from nblocks={GRIDS[0]}"
    # rejected before any launch: `out` overlapping the input (in place would race with the peers' loads) ...
    t = src.place(torch.ones(64, device="cuda"))
    for o in (t, src.buf[GUARD + 16:GUARD + 16 + 256].view(torch.float32)):
        try:
            comm.all_reduce_oneshot(t, o)
            raise AssertionError("an overlapping one-shot `out` was accepted")
        except ValueError:
            pass
    # ... and a range past the end of the heap
    out = torch.empty(64, device="cuda")
    rc = comm.lib.bnet_allreduce_oneshot(comm.h, comm.heap_bytes - 128, C.c_void_p(out.data_ptr()), 64, 0, 0, 1, 0,
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc < 0 and b"outside the heap" in comm.lib.bnet_coll_last_error(), "a one-shot range outside the heap was accepted"
    assert comm.status() == 0
    chk.report("oneshot")
    teardown()


def job_ll():
    """The barrier-free small-message kernel: odd counts in and out of place with guarded neighbours, different data on
    every call (a word left from an earlier call must not pass as current), the capacity limit, the `auto` dispatch at
    the limit and one step above it, and a captured CUDA graph replayed on new data."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(HEAP)
    cap = 4 * comm.ll_words                                         # bytes
    ibuf, obuf = Arena(comm, cap, heap=False), Arena(comm, cap, heap=False)
    chk = Checker()
    seed = 2000
    calls = 0
    for dtype in DTYPES:
        es = torch.empty((), dtype=dtype).element_size()
        for n in (1, 2, 3, 255, 256, 257, cap // es):
            for op in OPS:
                for inplace in (False, True):
                    seed += 1
                    xs = rank_inputs(seed, n, dtype)
                    x = ibuf.place(xs[RANK])
                    out = x if inplace else obuf.window(n, dtype)
                    comm.all_reduce_ll(x, None if inplace else out, op=op)
                    torch.cuda.synchronize()
                    calls += 1
                    what = f"ll {dtype} {op} n={n} {'in place' if inplace else 'out of place'}"
                    ibuf.check(what + " (input)")
                    if not inplace:
                        obuf.check(what + " (out)")
                        assert torch.equal(bits(x), bits(xs[RANK])), f"{what}: the input changed"
                    chk.check(out, xs, op, dtype, "ll", what)
                    assert same_on_every_rank(out), f"{what}: ranks hold different bits"
        # one element past the area: refused before any launch
        x = torch.zeros(cap // es + 1, dtype=dtype, device="cuda")
        try:
            comm.all_reduce_ll(x)
            raise AssertionError(f"ll {dtype}: a message one element past the LL area was accepted")
        except RuntimeError as e:
            assert "does not fit" in str(e), e
    # the `auto` dispatch of a heap tensor: at the LL capacity (LL), and the next multiple of 16 * W bytes above it
    # (two-shot, or the in-switch kernel from three ranks with multicast)
    big = (cap // (16 * WORLD) + 1) * 16 * WORLD
    heap = Arena(comm, big, heap=True)
    for nbytes, path in ((cap, "ll" if WORLD > 1 else "p2p"),
                         (big, "nvls" if comm.has_multicast and WORLD > 2 else "p2p")):
        for dtype in (torch.bfloat16, torch.float32):
            for op in ("sum", "avg"):
                seed += 1
                xs = rank_inputs(seed, nbytes // torch.empty((), dtype=dtype).element_size(), dtype)
                t = heap.place(xs[RANK])
                sync()
                comm.all_reduce(t, op)
                sync()
                what = f"auto {dtype} {op} {nbytes} bytes (expected path {path})"
                heap.check(what)
                chk.check(t, xs, op, dtype, path, what)
                assert same_on_every_rank(t), f"{what}: ranks hold different bits"
    # a captured LL call, replayed on new data every time
    n = 1000
    x = torch.zeros(n, device="cuda")
    y = torch.empty_like(x)
    sync()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        comm.all_reduce_ll(x, y)                                     # (warm-up outside the capture)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        comm.all_reduce_ll(x, y)
    for rep in range(6):
        seed += 1
        xs = rank_inputs(seed, n, torch.float32)
        x.copy_(xs[RANK])
        g.replay()
        torch.cuda.synchronize()
        chk.check(y, xs, "sum", torch.float32, "ll", f"ll graph replay {rep}")
    assert comm.status() == 0
    chk.report("ll")
    if RANK == 0:
        print(f"ll: {calls} consecutive calls with new data, dtypes and sizes mixed on one area; 6 graph replays", flush=True)
    teardown()


def job_nonfinite():
    """NaN and +-Inf inputs on every path.  sum / avg: a NaN on one rank, or +Inf with -Inf, gives NaN; +-Inf with finite
    values gives +-Inf; a finite 16-bit sum gives +-Inf exactly where the dtype's rounding of the float64 sum overflows.
    max / min: element for element what NCCL's all-reduce returns on the same tensors."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(HEAP)
    paths = ["p2p"] + (["nvls"] if comm.has_multicast else []) + ["oneshot", "ll"]
    chk = Checker()
    heap = Arena(comm, 16 * WORLD * (4 * 7 * 512 + 1), heap=True)
    dst = Arena(comm, 16 * WORLD * (4 * 7 * 512 + 1), heap=False)
    nccl_drops_nan = {}
    seed = 3000
    for dtype in DTYPES:
        for per in (25, 4 * 7 * 512 + 1):
            n = per * WORLD * elems(dtype)
            i = torch.arange(n, device="cuda")
            owner = (i // 8) % WORLD                       # the rank that holds an element's special value
            other = (owner + 1) % WORLD
            seed += 1
            base = [torch.randn(n, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed * 64 + r)).to(dtype)
                    for r in range(WORLD)]
            big = torch.finfo(dtype).max
            for op in OPS:
                xs = []
                for r in range(WORLD):
                    x = base[r].clone()
                    x[(i % 8 == 1) & (owner == r)] = float("nan")
                    x[(i % 8 == 2) & (owner == r)] = float("inf")
                    x[(i % 8 == 3) & (owner == r)] = -float("inf")
                    x[(i % 8 == 4) & (owner == r)] = float("inf")
                    if WORLD > 1:
                        x[(i % 8 == 4) & (other == r)] = -float("inf")
                    x[i % 8 == 7] = float("nan")                        # NaN on every rank
                    if op == "sum" and dtype != torch.float32:
                        # every rank 0.75 max: for W >= 2 the sum overflows the dtype; W / (W + 1) max: it does not
                        x[i % 16 == 5] = 0.75 * big
                        x[i % 16 == 13] = -0.75 * big
                        x[i % 16 == 6] = big / (WORLD + 1)
                    xs.append(x)
                X = torch.stack([x.double() for x in xs])
                nccl = None
                if op in ("max", "min"):
                    nccl = xs[RANK].clone()
                    sync()
                    dist.all_reduce(nccl, op=dist.ReduceOp.MAX if op == "max" else dist.ReduceOp.MIN)
                    torch.cuda.synchronize()
                    one_nan = (i % 8 == 1)
                    nccl_drops_nan[(dtype, op)] = not bool(nccl[one_nan].isnan().any()) if WORLD > 1 else None
                for path in paths:
                    if path == "ll" and n * xs[0].element_size() > 4 * comm.ll_words:
                        continue
                    what = f"{path} {dtype} {op} {per} vectors/rank with NaN/Inf"
                    if path == "oneshot":
                        t = heap.place(xs[RANK])
                        out = dst.window(n, dtype)
                        sync()
                        comm.all_reduce_oneshot(t, out, op)
                        sync()
                        dst.check(what)
                    elif path == "ll":
                        t = dst.place(xs[RANK])
                        out = comm.all_reduce_ll(t, op=op)
                        torch.cuda.synchronize()
                        dst.check(what)
                    else:
                        out = heap.place(xs[RANK])
                        sync()
                        comm.all_reduce(out, op, algo=path)
                        torch.cuda.synchronize()
                        heap.check(what)
                    assert same_on_every_rank(out), f"{what}: ranks hold different bits"
                    if op in ("max", "min"):
                        assert torch.equal(out.isnan(), nccl.isnan()), f"{what}: NaNs differ from NCCL's"
                        fin = ~nccl.isnan()
                        assert torch.equal(out[fin].double(), nccl[fin].double()), f"{what}: values differ from NCCL's"
                        continue
                    want = X.sum(0) if op == "sum" else X.sum(0) / WORLD
                    want_dt = want.to(dtype).double()               # NaN, +-Inf, and the dtype's overflow of the sum
                    got = out.double()
                    assert torch.equal(got.isnan(), want_dt.isnan()), f"{what}: NaN pattern differs from float64"
                    inf = want_dt.isinf()
                    assert torch.equal(got.isinf(), inf), f"{what}: Inf pattern differs from float64"
                    assert torch.equal(got[inf], want_dt[inf]), f"{what}: signs of the infinities differ"
                    fin = want_dt.isfinite()
                    chk.check(out[fin], [x[fin] for x in xs], op, dtype, path, what)
    assert comm.status() == 0
    chk.report("nonfinite")
    if RANK == 0:
        print(f"nonfinite: W={WORLD} paths {paths}; NCCL max/min with a NaN on one rank returns the number (NaN loses): "
              f"{ {str(k[0]).split('.')[-1] + ' ' + k[1]: v for k, v in nccl_drops_nan.items()} }", flush=True)
    teardown()


def job_pack_cast():
    """bnet_pack_cast for all five (source, destination) dtype pairs, bit for bit against (src.float() * scale).to(dst):
    explicit offsets with guarded gaps, an item longer than the 64-CTA grid stride, a scale that is not a power of two."""
    from bagua_net_b200.ops import pack_cast
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(64 << 20)
    scale = float(torch.tensor(0.3, dtype=torch.float32))            # (fp32, as the kernel multiplies)
    sizes = (1, 7, 1000, 64 * 256 * 3 + 13, 5)
    gap = 9
    for s_dt, d_dt in ((torch.float32, torch.bfloat16), (torch.bfloat16, torch.bfloat16), (torch.bfloat16, torch.float32),
                       (torch.float32, torch.float32), (torch.float16, torch.float32)):
        g = torch.Generator(device="cuda").manual_seed(5)
        ts = [(torch.randn(n, device="cuda", generator=g) * 100).to(s_dt) for n in sizes]
        offsets, o = [], gap
        for t in ts:
            offsets.append(o)
            o += t.numel() + gap
        dst = torch.full((o,), 12345.0, device="cuda").to(d_dt)
        sentinel = dst[0].clone()
        pack_cast(comm, ts, dst, offsets=offsets, scale=scale)
        torch.cuda.synchronize()
        covered = torch.zeros(o, dtype=torch.bool, device="cuda")
        for t, off in zip(ts, offsets):
            want = (t.float() * scale).to(d_dt)
            assert torch.equal(bits(dst[off:off + t.numel()]), bits(want)), f"pack_cast {s_dt}->{d_dt}: item of {t.numel()} differs"
            covered[off:off + t.numel()] = True
        assert bool((dst[~covered] == sentinel).all()), f"pack_cast {s_dt}->{d_dt}: a gap between items was written"
    print(f"rank {RANK}: pack_cast ok for f32->bf16, bf16->bf16, bf16->f32, f32->f32, f16->f32 (scale {scale})", flush=True)
    teardown()


JOBS = {k[4:]: v for k, v in globals().items() if k.startswith("job_")}

if __name__ == "__main__":
    JOBS[sys.argv[1]]()

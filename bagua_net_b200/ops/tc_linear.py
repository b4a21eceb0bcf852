"""Tensor-core (wgmma) linear layer and the fused row-parallel (GEMM + all-reduce) linear (csrc/cuda/tc_gemm.cu).

    y = tc_linear.linear(x, w, bias, relu=True)                # bf16 [M,K] x [N,K]^T -> bf16 [M,N], fused bias + ReLU
    y = tc_linear.row_parallel_linear(x_k, w_k, comm)          # every rank holds a K-shard; fp32 sum lands on EVERY rank
    y = tc_linear.linear_reduce_scatter(x_k, w_k, comm)        # ... or only on the rank that owns each row block
    y = tc_linear.allgather_linear(x_rows, w, comm)            # x sharded by rows: peers' shards are TMA-loaded over NVLink

The kernel stages operands with TMA (128-byte swizzle), multiplies with ``wgmma.mma_async`` into register accumulators
and applies the epilogue from there; ``row_parallel_linear`` is the "compute step followed by a collective in ONE kernel"
form: the epilogue adds its fp32 tile into every rank's symmetric-heap output (``multimem.red`` through the NVSwitch
multicast mapping, ``red.global`` per peer otherwise), so no separate all-reduce runs.

The reference has no compute path (SURVEY.md §2.6) — this belongs to the GPU side of the framework.

On by default (``BNET_TC=0`` disables); ``self_check()`` must pass on the GPU at hand before any caller trusts it
(``trusted()``), and every launch carries a device-side watchdog (``last_error()``)."""
from __future__ import annotations

import ctypes as C
import os

import torch

from ..utils.native import load

_lib = None
_err: dict[int, torch.Tensor] = {}
LAUNCHES = 0


class Plan(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("swap", "bn", "stages", "grid_x", "grid_y", "grid_z", "smem_bytes", "k_blocks",
                                       "k_per_split", "ctas")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


def _L():
    global _lib
    if _lib is None:
        _lib = load()
        vp, i = C.c_void_p, C.c_int
        _lib.bnet_tc_supported.restype = i
        _lib.bnet_tc_plan.argtypes = [i, i, i, i, i, C.POINTER(Plan)]
        _lib.bnet_tc_linear.argtypes = [vp, vp, vp, vp, i, i, i, i, i, i, i, vp, vp]
        _lib.bnet_tc_linear_reduce.argtypes = [vp, vp, vp, C.POINTER(vp), i, i, i, i, i, i, i, i, i, vp, vp]
        _lib.bnet_tc_linear_splitk.argtypes = [vp, vp, vp, vp, vp, vp, i, i, i, i, i, i, i, i, vp, vp]
        _lib.bnet_tc_linear_dgrad.argtypes = [vp, vp, vp, i, i, i, i, i, i, vp, vp]
        _lib.bnet_tc_linear_wgrad.argtypes = [vp, vp, vp, i, i, i, i, i, i, vp, vp]
        _lib.bnet_tc_allgather_linear.argtypes = [C.POINTER(vp), i, i, vp, vp, vp, i, i, i, i, i, i, vp, vp]
        _lib.bnet_tc_linear_reduce_scatter.argtypes = [vp, vp, vp, C.POINTER(vp), i, i, i, i, i, i, i, i, vp, vp]
        _lib.bnet_tc_last_error.restype = C.c_char_p
        _lib.bnet_tc_smem_desc.restype = C.c_uint64
        _lib.bnet_tc_smem_desc.argtypes = [C.c_uint32]
    return _lib


def enabled() -> bool:
    """Switch for callers (models, bench).  On by default (callers still wait for ``trusted()``); BNET_TC=0 keeps every
    linear layer on cuBLAS."""
    return os.environ.get("BNET_TC", "1") == "1"


def supported() -> bool:
    return torch.cuda.is_available() and bool(_L().bnet_tc_supported())


def plan(M: int, N: int, K: int, reduce: bool = False, splits: int = 1) -> dict:
    """The tiling the kernel would use (host-only; works without a GPU)."""
    p = Plan()
    if _L().bnet_tc_plan(M, N, K, 1 if reduce else 0, splits, C.byref(p)) != 0:
        raise ValueError(_L().bnet_tc_last_error().decode())
    return p.as_dict()


def _err_flag(dev: int) -> torch.Tensor:
    if dev not in _err:
        _err[dev] = torch.zeros(1, dtype=torch.int32, device=f"cuda:{dev}")
    return _err[dev]


def last_error(device: int | None = None) -> int:
    """Synchronises.  0 = every launch so far completed; 1/2/3 = the TMA producer / the MMA warpgroups / a split-K slice waiting for its turn gave up
    waiting (the watchdog turned a stuck pipeline into this code).  Reading clears it."""
    dev = torch.cuda.current_device() if device is None else device
    f = _err_flag(dev)
    v = int(f.item())
    if v:
        f.zero_()
    return v


def _check_operands(x, w, bias):
    if not (x.is_cuda and w.is_cuda and x.dtype == torch.bfloat16 and w.dtype == torch.bfloat16):
        raise TypeError("tc_linear needs bf16 CUDA tensors")
    if x.dim() != 2 or w.dim() != 2 or x.shape[1] != w.shape[1]:
        raise ValueError(f"shapes do not multiply: x {tuple(x.shape)} w {tuple(w.shape)}")
    if x.stride(1) != 1 or w.stride(1) != 1:
        raise ValueError("operands must be K-contiguous")
    if bias is not None and not (bias.is_cuda and bias.dtype == torch.bfloat16 and bias.is_contiguous()
                                 and bias.numel() == w.shape[0]):
        raise ValueError("bias must be a contiguous bf16 vector with one entry per output feature")


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _auto_splits(M: int, N: int, K: int) -> int:
    """Small-batch layers are weight streaming: with M <= 64 a [M, N] output has only N / 128 tiles — 32 CTAs for the VGG
    classifier — and one SM cannot pull its 128 x K weight slab at more than a fraction of HBM speed.  Splitting K over
    grid.z puts every SM to work; the partial tiles meet as fp32 adds in a small workspace."""
    if M > 64 or K < 2048:
        return 1
    tiles = (N + 127) // 128
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return max(1, min(8, sms // max(tiles, 1), K // 1024))


_scratch: dict = {}


def _splitk_scratch(device, M: int, N: int):
    """fp32 [M, N] workspace + one counter per output tile, shared by every split-K call of that shape on that device
    (calls on one stream are ordered; the kernel hands both back all-zero)."""
    key = (device.index, M, N)
    if key not in _scratch:
        tiles = ((N + 31) // 32) * ((M + 31) // 32) + 64        # upper bound on the tile count of any plan
        _scratch[key] = (torch.zeros((M, N), dtype=torch.float32, device=device),
                         torch.zeros(tiles, dtype=torch.int32, device=device))
    return _scratch[key]


def linear(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None, relu: bool = False,
           out: torch.Tensor | None = None, splits: int | None = None) -> torch.Tensor:
    """``act(x @ w.T + bias)`` on the wgmma tensor cores; x [M,K], w [N,K] (torch ``Linear.weight``), bf16.
    ``splits``: K slices (None = automatic, see ``_auto_splits``; 1 = one pass with the epilogue fused in the kernel)."""
    global LAUNCHES
    _check_operands(x, w, bias)
    M, K = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.bfloat16, device=x.device)
    assert out.dtype == torch.bfloat16 and out.shape == (M, N) and out.stride(1) == 1
    L = _L()
    if splits is None:
        splits = _auto_splits(M, N, K)
    if splits > 1:
        # split-K with the finish inside the kernel: the K slices add fp32 partial tiles into a workspace, the slice that
        # arrives last at a tile applies bias / ReLU, writes bf16 and re-zeroes what it read — ONE launch.  The workspace
        # and the tile counters are zero between calls by construction, so they are allocated (and cleared) once.
        ws, counters = _splitk_scratch(x.device, M, N)
        rc = L.bnet_tc_linear_splitk(x.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None, out.data_ptr(),
                                     ws.data_ptr(), counters.data_ptr(), M, N, K, x.stride(0), w.stride(0), out.stride(0),
                                     1 if relu else 0, splits, _err_flag(x.device.index).data_ptr(), _stream())
        if rc < 0:
            raise RuntimeError(f"bnet_tc_linear_splitk: {L.bnet_tc_last_error().decode()}")
        LAUNCHES += rc
        return out
    rc = L.bnet_tc_linear(x.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None, out.data_ptr(), M, N,
                          K, x.stride(0), w.stride(0), out.stride(0), 1 if relu else 0,
                          _err_flag(x.device.index).data_ptr(), _stream())
    if rc < 0:
        raise RuntimeError(f"bnet_tc_linear: {L.bnet_tc_last_error().decode()}")
    LAUNCHES += rc
    return out


def linear_dgrad(gy: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """``gy @ w`` (dX of a linear layer): gy [M,N], w [N,K] as stored — w is read MN-major, no transpose is made."""
    global LAUNCHES
    M, N = gy.shape
    K = w.shape[1]
    assert gy.dtype == w.dtype == torch.bfloat16 and w.shape[0] == N and gy.stride(1) == 1 and w.stride(1) == 1
    dx = torch.empty((M, K), dtype=torch.bfloat16, device=gy.device)
    L = _L()
    rc = L.bnet_tc_linear_dgrad(gy.data_ptr(), w.data_ptr(), dx.data_ptr(), M, N, K, gy.stride(0), w.stride(0), dx.stride(0),
                                _err_flag(gy.device.index).data_ptr(), _stream())
    if rc < 0:
        raise RuntimeError(f"bnet_tc_linear_dgrad: {L.bnet_tc_last_error().decode()}")
    LAUNCHES += rc
    return dx


def linear_wgrad(gy: torch.Tensor, x: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """``gy.T @ x`` (dW of a linear layer): gy [M,N], x [M,K] as stored — both read MN-major (the batch is the reduction).
    ``out``: a bf16 [N,K] tensor with unit inner stride and a 16-byte row pitch to write into (e.g. the parameter's slice of
    a training engine's flat gradient buffer)."""
    global LAUNCHES
    M, N = gy.shape
    K = x.shape[1]
    assert gy.dtype == x.dtype == torch.bfloat16 and x.shape[0] == M and gy.stride(1) == 1 and x.stride(1) == 1
    if out is not None and (tuple(out.shape) != (N, K) or out.dtype != torch.bfloat16 or out.stride(1) != 1 or out.stride(0) % 8
                            or out.data_ptr() % 16):
        out = None
    dw = torch.empty((N, K), dtype=torch.bfloat16, device=gy.device) if out is None else out
    L = _L()
    rc = L.bnet_tc_linear_wgrad(gy.data_ptr(), x.data_ptr(), dw.data_ptr(), M, N, K, gy.stride(0), x.stride(0), dw.stride(0),
                                _err_flag(gy.device.index).data_ptr(), _stream())
    if rc < 0:
        raise RuntimeError(f"bnet_tc_linear_wgrad: {L.bnet_tc_last_error().decode()}")
    LAUNCHES += rc
    return dw


def _bwd_on_tc(gy, x, w) -> bool:
    """The backward GEMMs run on the wgmma kernel too (BNET_TC_BWD=0 keeps them on cuBLAS) when the operands meet the
    TMA constraints: 16-byte row pitches, and more than 64 output features for dW."""
    if os.environ.get("BNET_TC_BWD", "1") != "1":
        return False
    N, K = w.shape
    return (gy.is_contiguous() and N > 64 and N % 8 == 0 and K % 8 == 0 and x.stride(1) == 1 and x.stride(0) % 8 == 0
            and w.stride(1) == 1 and w.stride(0) % 8 == 0)


def weight_grad(gy: torch.Tensor, x: torch.Tensor, w: torch.Tensor, tc: bool) -> torch.Tensor:
    """dW = gy.T @ x of a linear layer.  When a training engine registered a gradient slice for `w` (ops/grad_target.py) the
    GEMM writes straight into it — the wgmma kernel through its output pointer, cuBLAS through ``out=`` — and the slice is
    handed to autograd for adoption: no tensor of its own, no accumulate pass over the (for VGG16's fc1: 205 MB) gradient."""
    from . import grad_target

    dst = grad_target.lookup(w, shape=(gy.shape[1], x.shape[1]), dtype=gy.dtype)
    if dst is not None and not dst.is_contiguous():
        dst = None
    if tc:
        gw = linear_wgrad(gy, x, out=dst)
        return grad_target.adopt(dst) if dst is not None and gw.data_ptr() == dst.data_ptr() else gw
    if dst is not None:
        torch.mm(gy.t(), x, out=dst)
        return grad_target.adopt(dst)
    return gy.t() @ x


class _LinearAct(torch.autograd.Function):
    """Forward on the wgmma kernel (bias and ReLU in its epilogue); dX and dW on the same kernel with MN-major
    operands (no transposed copies), or on cuBLAS when the shapes do not meet the TMA constraints."""

    @staticmethod
    def forward(ctx, x, w, bias, relu):
        y = linear(x, w, bias, relu)
        ctx.relu = relu
        ctx.has_bias = bias is not None
        ctx.save_for_backward(x, w, y if relu else None)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w, y = ctx.saved_tensors
        if ctx.relu:
            gy = gy * (y > 0).to(gy.dtype)
        gy = gy.contiguous()
        tc = _bwd_on_tc(gy, x, w)
        gx = gw = None
        if ctx.needs_input_grad[0]:
            gx = linear_dgrad(gy, w) if tc else gy @ w
        if ctx.needs_input_grad[1]:
            gw = weight_grad(gy, x, w, tc)
        gb = gy.sum(0) if ctx.has_bias and ctx.needs_input_grad[2] else None
        return gx, gw, gb, None


def linear_bias_act(x, w, bias=None, relu=False):
    """Autograd-aware ``linear``."""
    return _LinearAct.apply(x, w, bias, relu)


_trusted: bool | None = None


LAST_CHECK_DEFINITIVE = True      # did the last child-process check end with a verdict (False: timeout / could not run)?


def _isolated_self_check(timeout: float = 180.0, check: str | None = None, tag: str = "tc_self_check") -> bool:
    """``self_check()`` (or `check`: Python source that leaves its verdict in ``ok``) in a child process: a kernel that
    faults (a poisoned CUDA context) or hangs past its own watchdog must not take the training process with it.  The verdict is cached per (library build, GPU model) under
    ``$BNET_CACHE_DIR`` (default ``~/.cache/bnet``), so only the first process on a machine pays for it."""
    import hashlib
    import json
    import subprocess
    import sys

    from .. import LIB_DIR, LIB_NAME, REPO_ROOT

    lib = os.path.join(LIB_DIR, LIB_NAME)
    try:
        key = f"{os.path.getmtime(lib):.0f}-{os.path.getsize(lib)}-{torch.cuda.get_device_name()}-{torch.version.cuda}"
    except Exception:  # noqa: BLE001
        return False
    cache_dir = os.environ.get("BNET_CACHE_DIR") or os.path.join(os.path.expanduser("~"), ".cache", "bnet")
    path = os.path.join(cache_dir, tag + "_" + hashlib.sha1(key.encode()).hexdigest()[:16] + ".json")
    global LAST_CHECK_DEFINITIVE
    try:
        with open(path) as f:
            ok = bool(json.load(f)["ok"])
        LAST_CHECK_DEFINITIVE = True
        return ok
    except Exception:  # noqa: BLE001 — no verdict yet
        pass
    env = dict(os.environ, PYTHONPATH=REPO_ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""),
               CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", ""))
    if not env["CUDA_VISIBLE_DEVICES"]:
        env.pop("CUDA_VISIBLE_DEVICES")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):     # the child is a plain 1-GPU process
        env.pop(k, None)
    body = check or "from bagua_net_b200.ops import tc_linear; ok = tc_linear.self_check()"
    code = "import sys, torch; torch.cuda.set_device(%d); %s; sys.exit(0 if ok else 3)" % (torch.cuda.current_device(), body)
    try:
        rc = subprocess.run([sys.executable, "-c", code], env=env, timeout=timeout, stdout=subprocess.DEVNULL,
                            stderr=subprocess.DEVNULL).returncode
    except Exception:  # noqa: BLE001 — timeout, spawn failure
        rc = None
    # exit 0 / 3: the check ran and passed / failed; death by a signal: a faulting kernel — all definitive, cached.  Anything
    # else (timeout under a profiler, no GPU for the child, an import problem) is no verdict: not trusted now, asked again
    # next time
    LAST_CHECK_DEFINITIVE = not (rc is None or (rc > 0 and rc != 3))
    if not LAST_CHECK_DEFINITIVE:
        return False
    ok = rc == 0
    try:
        os.makedirs(cache_dir, exist_ok=True)
        tmp = f"{path}.{os.getpid()}"
        with open(tmp, "w") as f:
            json.dump({"ok": ok, "key": key}, f)
        os.replace(tmp, path)
    except OSError:
        pass
    return ok


def trusted() -> bool:
    """enabled() and a passing self-check on this GPU, evaluated once per process.  The check runs in this process (about
    a second; every wait in the kernel carries a watchdog, so a wrong pipeline is an error code, not a hang);
    ``BNET_TC_ISOLATED_CHECK=1`` runs it in a child process instead (fault isolation, verdict cached per build and GPU)."""
    global _trusted
    if _trusted is None:
        if not (enabled() and supported()):
            _trusted = False
        elif os.environ.get("BNET_TC_ISOLATED_CHECK") == "1":
            _trusted = _isolated_self_check()
        else:
            if torch.cuda.is_current_stream_capturing():
                return False            # (not decided yet, and a capture is no place to decide)
            _trusted = self_check()
    return _trusted


class TCLinear(torch.nn.Linear):
    """``nn.Linear`` (same parameters, same state_dict keys) with an optional fused ReLU whose forward runs on the
    wgmma kernel when ``BNET_TC=1`` and the self-check passed on this GPU; cuBLAS + eager ReLU otherwise."""

    def __init__(self, in_features, out_features, bias=True, relu=False, **kw):
        super().__init__(in_features, out_features, bias=bias, **kw)
        self.relu = relu

    def forward(self, x):
        if (x.is_cuda and x.dtype == torch.bfloat16 and self.weight.dtype == torch.bfloat16 and x.dim() == 2
                and x.stride(1) == 1 and self.in_features % 8 == 0 and x.stride(0) % 8 == 0 and trusted()):
            return linear_bias_act(x, self.weight, self.bias, self.relu)
        y = torch.nn.functional.linear(x, self.weight, self.bias)
        return torch.relu(y) if self.relu else y

    def extra_repr(self):
        return super().extra_repr() + f", relu={self.relu}, wgmma={'on' if enabled() else 'off'}"


def row_parallel_linear(x: torch.Tensor, w: torch.Tensor, comm, bias: torch.Tensor | None = None,
                        out: torch.Tensor | None = None, splits: int = 1) -> torch.Tensor:
    """Row-parallel linear: rank r holds x[:, K_r] and w[:, K_r]; returns fp32 ``sum_r x_r @ w_r.T (+ bias)`` on every
    rank, produced by ONE kernel per rank whose epilogue adds into all ranks' outputs over NVLink.

    ``out`` must come from ``comm.alloc`` (same offset on every rank); pass it back in to reuse the buffer.  Two rank
    barriers bracket the kernel: outputs are zero before anyone adds, and all adds have landed before anyone reads."""
    global LAUNCHES
    _check_operands(x, w, bias)
    M, K = x.shape
    N = w.shape[0]
    if out is None:
        out = comm.alloc(M * N, torch.float32).view(M, N)
    assert out.dtype == torch.float32 and out.shape == (M, N) and out.is_contiguous()
    off = comm.offset_of(out)
    out.zero_()
    comm.barrier()
    if comm.world > 1 and comm.has_multicast:
        ptrs, mc = [int(comm.lib.bnet_coll_mc_heap(comm.h)) + off], 1
    else:
        ptrs = [int(comm.lib.bnet_coll_peer_heap(comm.h, r)) + off if r != comm.rank else out.data_ptr()
                for r in range(comm.world)]
        mc = 0
    arr = (C.c_void_p * len(ptrs))(*ptrs)
    L = _L()
    b = bias if (bias is not None and comm.rank == 0) else None       # added once, not once per rank
    rc = L.bnet_tc_linear_reduce(x.data_ptr(), w.data_ptr(), b.data_ptr() if b is not None else None, arr, len(ptrs), mc,
                                 M, N, K, x.stride(0), w.stride(0), out.stride(0), splits,
                                 _err_flag(x.device.index).data_ptr(), _stream())
    if rc < 0:
        raise RuntimeError(f"bnet_tc_linear_reduce: {L.bnet_tc_last_error().decode()}")
    LAUNCHES += rc
    comm.barrier()
    return out


def _peer_ptrs(comm, t):
    off = comm.offset_of(t)
    return [int(comm.lib.bnet_coll_peer_heap(comm.h, r)) + off if r != comm.rank else t.data_ptr() for r in range(comm.world)]


def allgather_linear(x_shard: torch.Tensor, w: torch.Tensor, comm, bias: torch.Tensor | None = None, relu: bool = False,
                     sync: bool = True) -> torch.Tensor:
    """``act(all_gather(x_shard) @ w.T + bias)`` in ONE kernel: x is sharded by rows over the ranks (sequence / batch
    parallel input of a column-parallel layer); ``x_shard`` [rows, K] must come from ``comm.alloc`` (same offset on every
    rank) with rows a multiple of 128.  Each tile's operand is loaded by TMA straight from the owning rank's memory over
    NVLink — the gathered activation is never materialised.  Returns bf16 [world * rows, N].
    ``sync``: rank barriers before (every shard is written) and after (nobody overwrites a shard still being read)."""
    global LAUNCHES
    _check_operands(x_shard, w, bias)
    rows, K = x_shard.shape
    N = w.shape[0]
    ptrs = _peer_ptrs(comm, x_shard)
    out = torch.empty((rows * comm.world, N), dtype=torch.bfloat16, device=x_shard.device)
    if sync:
        comm.barrier()
    arr = (C.c_void_p * len(ptrs))(*ptrs)
    L = _L()
    rc = L.bnet_tc_allgather_linear(arr, len(ptrs), rows, w.data_ptr(), bias.data_ptr() if bias is not None else None,
                                    out.data_ptr(), N, K, x_shard.stride(0), w.stride(0), out.stride(0), 1 if relu else 0,
                                    _err_flag(x_shard.device.index).data_ptr(), _stream())
    if rc < 0:
        raise RuntimeError(f"bnet_tc_allgather_linear: {L.bnet_tc_last_error().decode()}")
    LAUNCHES += rc
    if sync:
        comm.barrier()
    return out


def linear_reduce_scatter(x: torch.Tensor, w: torch.Tensor, comm, bias: torch.Tensor | None = None,
                          out: torch.Tensor | None = None, splits: int = 1) -> torch.Tensor:
    """Row-parallel linear whose result stays sharded: rank r ends up with rows [r*M/world, (r+1)*M/world) of
    ``sum_r x_r @ w_r.T (+ bias)`` as fp32 [M / world, N].  ONE kernel per rank: every output tile is added straight into
    its owner's symmetric-heap buffer (``red.global.add.v4.f32`` over NVLink) — GEMM -> reduce-scatter fused."""
    global LAUNCHES
    _check_operands(x, w, bias)
    M, K = x.shape
    N = w.shape[0]
    if M % comm.world:
        raise ValueError("the batch must divide by the number of ranks")
    if out is None:
        out = comm.alloc(M // comm.world * N, torch.float32).view(M // comm.world, N)
    assert out.dtype == torch.float32 and out.shape == (M // comm.world, N) and out.is_contiguous()
    ptrs = _peer_ptrs(comm, out)
    out.zero_()
    comm.barrier()
    arr = (C.c_void_p * len(ptrs))(*ptrs)
    L = _L()
    b = bias if (bias is not None and comm.rank == 0) else None
    rc = L.bnet_tc_linear_reduce_scatter(x.data_ptr(), w.data_ptr(), b.data_ptr() if b is not None else None, arr, len(ptrs),
                                         M, N, K, x.stride(0), w.stride(0), out.stride(0), splits,
                                         _err_flag(x.device.index).data_ptr(), _stream())
    if rc < 0:
        raise RuntimeError(f"bnet_tc_linear_reduce_scatter: {L.bnet_tc_last_error().decode()}")
    LAUNCHES += rc
    comm.barrier()
    return out


def self_check(verbose: bool = False) -> bool:
    """Run the kernel on a few shapes (both operand orientations, ragged M/N/K, bias, ReLU) against an fp32 PyTorch
    reference.  False — never an exception — when it is unsupported, errs, trips the watchdog or is numerically off."""
    try:
        if not supported():
            return False
        g = torch.Generator(device="cuda").manual_seed(7)
        # (the last shape is a small-batch, long-K layer: the automatic split-K path; the others run the fused epilogue)
        for (M, N, K, relu) in [(32, 256, 512, True), (48, 200, 264, False), (256, 384, 1024, True), (130, 136, 72, False),
                                (32, 512, 4096, True)]:
            x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
            w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
            b = torch.randn(N, device="cuda", generator=g).bfloat16()
            y = linear(x, w, b, relu, splits=None if K >= 4096 else 1)
            if last_error():
                return False
            ref = x.float() @ w.float().t() + b.float()
            if relu:
                ref = torch.relu(ref)
            err = (y.float() - ref).abs().max().item()
            if verbose:
                print(f"tc_linear {M}x{N}x{K} relu={relu}: max abs err {err:.4f}")
            if not (err < 0.06):
                return False
            if N > 64 and os.environ.get("BNET_TC_BWD", "1") == "1":       # the backward GEMMs (MN-major operands)
                gy = torch.randn(M, N, device="cuda", generator=g).bfloat16()
                dx, dw = linear_dgrad(gy, w), linear_wgrad(gy, x)
                if last_error():
                    return False
                e1 = (dx.float() - gy.float() @ w.float()).abs().max().item()
                rdw = gy.float().t() @ x.float()
                e2 = ((dw.float() - rdw).abs().max() / rdw.abs().max().clamp_min(1e-6)).item()
                if verbose:
                    print(f"tc_linear dgrad max abs err {e1:.4f}, wgrad max rel err {e2:.4f}")
                if not (e1 < 0.1 and e2 < 0.02):
                    return False
        return True
    except Exception as e:  # noqa: BLE001 — the caller falls back to cuBLAS
        if verbose:
            print(f"tc_linear self-check failed: {e!r}")
        return False

"""SymmComm — symmetric-memory communicator over the native bnet collectives.

One process per GPU.  Every rank allocates the same-sized heap with the CUDA VMM API,
the allocations are exchanged as POSIX fds and mapped into every peer (NVLink P2P), and —
when the fabric exposes it — bound to one multicast object so that the sm_90a kernels
can reduce inside the NVSwitch (multimem.ld_reduce) and broadcast through it
(multimem.st).  ``torch.distributed`` is only the control plane that carries the
128-byte handshake blobs (csrc/cuda/coll.cu, include/bnet/bnet_coll.h).

This is the intra-box data path the reference does not have: it is a TCP-only,
host-memory transport (reference: nthread_per_socket_backend.rs:252) that leaves the
reduction to NCCL's kernels.
"""
from __future__ import annotations

import ctypes as C
import os

import torch
import torch.distributed as dist

from ..utils.native import load

DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
OPS = {"sum": 0, "avg": 1, "max": 2, "min": 3}
ALGOS = {"auto": 0, "nvls": 1, "p2p": 2, "oneshot": 3, "ll": 0}
BLOB = 128
CLIP_ROW = 304          # doubles per bucket in the clipped step's partial rows (BNET_COLL_CLIP_ROW)
LARS_CHUNK = 4096       # vectors per norm slot of the LARS norm pass (BNET_LARS_CHUNK)
GROUPS_MAX = 64         # parameter groups of one engine, its default group included (BNET_GROUPS_MAX)


def check_lars_segments(table, shard_vecs: int, ntensors: int) -> int:
    """Validate a LARS segment table (rows {vec0, nvec, tensor, slot0}, see include/bnet/bnet_coll.h) for a shard of
    `shard_vecs` 16-byte vectors before it goes to the device, where the kernels trust it: sorted, in range, covering the
    shard exactly once, tensor indices below `ntensors`, slot0 the running count of BNET_LARS_CHUNK chunks.  Returns the
    number of norm slots; raises ValueError."""
    rows = [tuple(int(v) for v in r) for r in torch.as_tensor(table).reshape(-1, 4).tolist()]
    if not rows:
        raise ValueError("LARS segment table is empty")
    if not 0 < shard_vecs < 2 ** 31:
        raise ValueError(f"LARS shard of {shard_vecs} vectors is out of range")
    pos, slots = 0, 0
    for k, (vec0, nvec, tensor, slot0) in enumerate(rows):
        if vec0 != pos or nvec < 1 or pos + nvec > shard_vecs:
            raise ValueError(f"LARS segment {k} ({vec0}, {nvec}) does not continue the cover of the shard at vector {pos}")
        if not 0 <= tensor < ntensors:
            raise ValueError(f"LARS segment {k} names tensor {tensor} of {ntensors}")
        if slot0 != slots:
            raise ValueError(f"LARS segment {k} starts at slot {slot0}, expected {slots}")
        pos += nvec
        slots += (nvec + LARS_CHUNK - 1) // LARS_CHUNK
    if pos != shard_vecs:
        raise ValueError(f"LARS segments cover {pos} of the shard's {shard_vecs} vectors")
    return slots


def check_group_segments(table, shard_vecs: int, ngroups: int) -> None:
    """Validate a parameter-group segment table (rows {vec0, nvec, group, reserved}, see include/bnet/bnet_coll.h) for a
    shard of `shard_vecs` 16-byte vectors before it goes to the device, where the kernels trust it: sorted, covering the
    shard exactly once, group indices below `ngroups` (1..GROUPS_MAX).  Raises ValueError."""
    rows = [tuple(int(v) for v in r) for r in torch.as_tensor(table).reshape(-1, 4).tolist()]
    if not rows:
        raise ValueError("group segment table is empty")
    if not 0 < shard_vecs < 2 ** 31:
        raise ValueError(f"group shard of {shard_vecs} vectors is out of range")
    if not 1 <= ngroups <= GROUPS_MAX:
        raise ValueError(f"{ngroups} parameter groups: the kernels take 1..{GROUPS_MAX}")
    pos = 0
    for k, (vec0, nvec, group, _) in enumerate(rows):
        if vec0 != pos or nvec < 1 or pos + nvec > shard_vecs:
            raise ValueError(f"group segment {k} ({vec0}, {nvec}) does not continue the cover of the shard at vector {pos}")
        if not 0 <= group < ngroups:
            raise ValueError(f"group segment {k} names group {group} of {ngroups}")
        pos += nvec
    if pos != shard_vecs:
        raise ValueError(f"group segments cover {pos} of the shard's {shard_vecs} vectors")


def check_lars_tensors(table, nslots: int) -> None:
    """Validate a LARS tensor table (rows {slot0, nslots, excluded, reserved}): every slot range inside `nslots`."""
    rows = torch.as_tensor(table).reshape(-1, 4).tolist()
    if not rows:
        raise ValueError("LARS tensor table is empty")
    for j, (slot0, n, _, _) in enumerate(rows):
        if n < 0 or slot0 < 0 or slot0 + n > nslots:
            raise ValueError(f"LARS tensor {j}: slots [{slot0}, {slot0 + n}) outside the {nslots} slots")


def _host_identity():
    import socket

    try:
        with open("/proc/sys/kernel/random/boot_id") as f:
            boot = f.read().strip()
    except OSError:
        boot = ""
    return socket.gethostname(), boot


class _CudaView:
    """Minimal __cuda_array_interface__ carrier so torch can wrap native memory zero-copy."""

    def __init__(self, ptr: int, nbytes: int, owner):
        self.__cuda_array_interface__ = {
            "shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None,
        }
        self._owner = owner


def _declare(lib):
    vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
    lib.bnet_coll_create.argtypes = [i, i, i, sz, C.POINTER(vp)]
    lib.bnet_coll_export.argtypes = [vp, C.c_char_p]
    lib.bnet_coll_import.argtypes = [vp, C.c_char_p]
    lib.bnet_coll_mc_add_device.argtypes = [vp]
    lib.bnet_coll_mc_bind.argtypes = [vp]
    lib.bnet_coll_destroy.argtypes = [vp]
    lib.bnet_coll_heap.restype = vp
    lib.bnet_coll_heap.argtypes = [vp]
    lib.bnet_coll_heap_bytes.restype = sz
    lib.bnet_coll_heap_bytes.argtypes = [vp]
    lib.bnet_coll_peer_heap.restype = vp
    lib.bnet_coll_peer_heap.argtypes = [vp, i]
    lib.bnet_coll_mc_heap.restype = vp
    lib.bnet_coll_mc_heap.argtypes = [vp]
    lib.bnet_coll_has_multicast.argtypes = [vp]
    lib.bnet_coll_status.restype = C.c_uint
    lib.bnet_coll_status.argtypes = [vp]
    lib.bnet_coll_last_error.restype = C.c_char_p
    lib.bnet_allreduce.argtypes = [vp, sz, sz, i, i, i, i, i, vp]
    lib.bnet_allreduce_oneshot.argtypes = [vp, sz, vp, sz, i, i, i, i, vp]
    lib.bnet_barrier.argtypes = [vp, i, vp]
    lib.bnet_allreduce_ll.argtypes = [vp, sz, sz, vp, vp, sz, i, i, vp]
    lib.bnet_allreduce_ll_area_bytes.restype = sz
    lib.bnet_allreduce_ll_area_bytes.argtypes = [i, sz]
    lib.bnet_fused_allreduce_sgd.argtypes = [vp, sz, sz, sz, i, C.c_float, C.c_float, C.c_float, C.c_float, vp, vp,
                                             i, i, i, vp]
    lib.bnet_fused_allreduce_sgd_hp.argtypes = [vp, sz, sz, sz, i, vp, vp, vp, i, i, i, vp]
    lib.bnet_fused_allreduce_adamw.argtypes = [vp, sz, sz, sz, i, vp, vp, vp, vp, i, i, i, vp]
    lib.bnet_fused_clip_reduce_norm.argtypes = [vp, sz, sz, i, vp, vp, i, i, vp]
    lib.bnet_fused_accum_reduce_norm.argtypes = [vp, sz, sz, i, vp, vp, i, i, vp]
    lib.bnet_fused_clip_coef.argtypes = [vp, vp, i, sz, C.c_float, vp, i, vp]
    lib.bnet_fused_clip_apply_sgd.argtypes = [vp, sz, sz, i, vp, vp, C.c_float, C.c_float, C.c_float, C.c_float, vp, vp, i, i, vp]
    lib.bnet_fused_clip_apply_sgd_hp.argtypes = [vp, sz, sz, i, vp, vp, vp, vp, vp, i, i, vp]
    lib.bnet_fused_clip_apply_adamw.argtypes = [vp, sz, sz, i, vp, vp, vp, vp, vp, vp, i, i, vp]
    lib.bnet_fused_lars_norm.argtypes = [vp, sz, i, vp, vp, vp, i, vp, i, i, vp]
    lib.bnet_fused_lars_trust.argtypes = [vp, vp, vp, i, sz, vp, vp, vp, vp, i, vp]
    lib.bnet_fused_lars_apply.argtypes = [vp, sz, sz, i, vp, vp, i, vp, vp, vp, vp, i, i, vp]
    lib.bnet_fused_allreduce_sgd_groups.argtypes = [vp, sz, sz, sz, i, vp, vp, i, vp, i, vp, vp, i, i, i, vp]
    lib.bnet_fused_allreduce_adamw_groups.argtypes = [vp, sz, sz, sz, i, vp, vp, i, vp, i, vp, vp, vp, i, i, i, vp]
    lib.bnet_fused_clip_apply_sgd_groups.argtypes = [vp, sz, sz, i, vp, vp, vp, vp, i, vp, i, vp, vp, i, i, vp]
    lib.bnet_fused_clip_apply_adamw_groups.argtypes = [vp, sz, sz, i, vp, vp, vp, vp, i, vp, i, vp, vp, vp, i, i, vp]
    lib.bnet_ema_update.argtypes = [vp, sz, vp, vp, vp, i, vp]
    lib.bnet_ema_advance.argtypes = [vp, vp, vp]
    lib.bnet_pack_cast.argtypes = [vp, i, vp, i, i, C.c_float, C.c_uint64, vp]


class SymmComm:
    """Symmetric heap + kernels.  ``group`` defaults to the world group; without an initialised
    process group the communicator is single-rank (the fused kernels still run — no peers)."""

    def __init__(self, heap_bytes: int, device: int | None = None, group=None):
        if not torch.cuda.is_available():
            raise RuntimeError("bagua_net_b200 collectives need a CUDA device (sm_90a); none is visible")
        self.lib = load()
        _declare(self.lib)
        self.group = group
        if dist.is_available() and dist.is_initialized():
            self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        else:
            self.rank, self.world = 0, 1
        self.device = torch.cuda.current_device() if device is None else device
        torch.cuda.set_device(self.device)
        self.launches = 0          # number of OUR kernels launched through this communicator
        h = C.c_void_p()
        self._chk(self.lib.bnet_coll_create(self.rank, self.world, self.device, heap_bytes, C.byref(h)), "create")
        self.h = h
        if self.world > 1:
            # the heap is shared through POSIX fds over a unix socket and mapped over NVLink: one host only
            hosts = [None] * self.world
            dist.all_gather_object(hosts, _host_identity(), group=group)
            if len(set(hosts)) > 1:
                raise RuntimeError("SymmComm needs all ranks of the group on ONE host (NVLink/NVSwitch domain); this group "
                                   f"spans {sorted(set(h[0] for h in hosts))}. Use one SymmComm per host and torch.distributed "
                                   "/ NCCL (optionally over the bnet plugin's TCP transport) between hosts.")
            blob = C.create_string_buffer(BLOB)
            self._chk(self.lib.bnet_coll_export(self.h, blob), "export")
            blobs = [None] * self.world
            dist.all_gather_object(blobs, bytes(blob.raw), group=group)
            self._chk(self.lib.bnet_coll_import(self.h, b"".join(blobs)), "import")
            # multicast: every rank must reach the same verdict before binding
            ok = self.lib.bnet_coll_mc_add_device(self.h) == 0
            ok = self._agree(ok)
            if ok:
                ok = self.lib.bnet_coll_mc_bind(self.h) == 0
                ok = self._agree(ok)
            if not ok and self.lib.bnet_coll_has_multicast(self.h):
                raise RuntimeError("ranks disagree on multicast availability")
            dist.barrier(group=group)
        self.heap_bytes = int(self.lib.bnet_coll_heap_bytes(self.h))
        self.heap_ptr = int(self.lib.bnet_coll_heap(self.h))
        self.has_multicast = bool(self.lib.bnet_coll_has_multicast(self.h))
        self._heap = torch.as_tensor(_CudaView(self.heap_ptr, self.heap_bytes, self), device=f"cuda:{self.device}")
        self._bump = 0
        self._lars_tables = {}     # device address of every validated LARS table -> (kind, rows, shard vectors or slots)
        self._group_tables = {}    # device address of every validated group segment table -> (rows, shard vectors, groups)
        # area of the barrier-free small-message all-reduce ("LL": the flag travels inside every 8-byte word)
        self.ll_words = int(os.environ.get("BNET_LL_WORDS", "8192"))          # 32 KiB of payload per rank and call
        area = int(self.lib.bnet_allreduce_ll_area_bytes(self.world, self.ll_words))
        self._ll = None
        if area + (1 << 20) <= self.heap_bytes:
            self._ll = self.alloc(area, torch.uint8)
            self._ll.zero_()
            torch.cuda.synchronize(self.device)
            if self.world > 1:
                dist.barrier(group=group)          # nobody pushes into an area that is still being cleared

    # ------------------------------------------------------------------ plumbing
    def _chk(self, rc, what):
        if rc is not None and rc < 0:
            raise RuntimeError(f"bnet coll {what} failed: {self.lib.bnet_coll_last_error().decode()}")
        return rc

    def _agree(self, ok: bool) -> bool:
        t = torch.tensor([1 if ok else 0], dtype=torch.int32, device=f"cuda:{self.device}")
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=self.group)
        return bool(t.item())

    def close(self):
        if getattr(self, "h", None):
            torch.cuda.synchronize(self.device)
            self._heap = None
            self.lib.bnet_coll_destroy(self.h)
            self.h = None

    def status(self) -> int:
        """0 = healthy; non-zero after a device-side watchdog trip (a peer never arrived)."""
        return int(self.lib.bnet_coll_status(self.h))

    # ------------------------------------------------------------------ heap tensors
    def alloc(self, numel: int, dtype: torch.dtype, align: int = 256) -> torch.Tensor:
        """Bump-allocate a tensor inside the symmetric heap (same offset on every rank when every
        rank performs the same sequence of calls)."""
        es = torch.empty((), dtype=dtype).element_size()
        # keep every allocation a whole number of 16-byte vectors per rank
        quantum = max(align, 16 * self.world)
        off = (self._bump + quantum - 1) // quantum * quantum
        nbytes = (numel * es + quantum - 1) // quantum * quantum
        if off + nbytes > self.heap_bytes:
            raise MemoryError(f"symmetric heap exhausted: need {off + nbytes} of {self.heap_bytes} bytes")
        self._bump = off + nbytes
        return self._heap[off:off + numel * es].view(dtype)

    def offset_of(self, t: torch.Tensor) -> int:
        off = t.data_ptr() - self.heap_ptr
        if off < 0 or off + t.numel() * t.element_size() > self.heap_bytes:
            raise ValueError("tensor does not live in the symmetric heap; use comm.alloc()")
        return off

    def peer_tensor(self, t: torch.Tensor, peer: int) -> torch.Tensor:
        """The same heap range as ``t`` on another rank (NVLink peer mapping)."""
        base = int(self.lib.bnet_coll_peer_heap(self.h, peer))
        nbytes = t.numel() * t.element_size()
        v = torch.as_tensor(_CudaView(base + self.offset_of(t), nbytes, self), device=f"cuda:{self.device}")
        return v.view(t.dtype).view(t.shape)

    # ------------------------------------------------------------------ collectives
    def _stream(self, stream):
        s = stream if stream is not None else torch.cuda.current_stream(self.device)
        return C.c_void_p(s.cuda_stream)

    def all_reduce(self, t: torch.Tensor, op: str = "sum", algo: str = "auto", channel: int = 1, nblocks: int = 0,
                   stream=None) -> torch.Tensor:
        """In-place all-reduce of a heap tensor.  numel*elsize must be a multiple of 16*world.
        ``algo="auto"`` sends messages that fit the LL area (<= 32 KiB by default) down the barrier-free path."""
        if algo in ("auto", "ll") and self._ll is not None and t.numel() * t.element_size() <= 4 * self.ll_words and self.world > 1:
            return self.all_reduce_ll(t, op=op, stream=stream)
        if algo == "ll":
            raise ValueError("message too large for the LL all-reduce")
        n = self._chk(self.lib.bnet_allreduce(self.h, self.offset_of(t), t.numel(), DT[t.dtype], OPS[op], ALGOS[algo],
                                              channel, nblocks, self._stream(stream)), "all_reduce")
        self.launches += n
        return t

    def all_reduce_oneshot(self, t: torch.Tensor, out: torch.Tensor, op: str = "sum", channel: int = 1,
                           nblocks: int = 0, stream=None) -> torch.Tensor:
        """Out-of-place all-reduce: every rank reads every rank's heap tensor ``t`` and writes the result to its own
        ``out`` (any CUDA memory).  ``out`` must not overlap ``t``: peers may still be reading ``t`` while this rank
        writes ``out``."""
        assert out.is_contiguous() and out.numel() == t.numel() and out.dtype == t.dtype
        nbytes = t.numel() * t.element_size()
        if out.data_ptr() < t.data_ptr() + nbytes and t.data_ptr() < out.data_ptr() + nbytes:
            raise ValueError("all_reduce_oneshot is out of place: `out` overlaps `t`, which the peers are still reading")
        n = self._chk(self.lib.bnet_allreduce_oneshot(self.h, self.offset_of(t), C.c_void_p(out.data_ptr()), t.numel(),
                                                      DT[t.dtype], OPS[op], channel, nblocks, self._stream(stream)),
                      "all_reduce_oneshot")
        self.launches += n
        return out

    def all_reduce_ll(self, t: torch.Tensor, out: torch.Tensor | None = None, op: str = "sum", stream=None) -> torch.Tensor:
        """Small-message all-reduce without a barrier: every rank pushes (payload, call number) words straight into every
        peer's receive area and sums what arrives — about one NVLink store latency.  ``t`` / ``out`` are ordinary CUDA
        tensors (``out`` defaults to ``t``: in place), at most ``4 * ll_words`` bytes; every rank must issue the same
        sequence of calls."""
        if self._ll is None:
            raise RuntimeError("the symmetric heap is too small for the LL area")
        out = t if out is None else out
        assert t.is_contiguous() and out.is_contiguous() and out.numel() == t.numel() and out.dtype == t.dtype
        n = self._chk(self.lib.bnet_allreduce_ll(self.h, self.offset_of(self._ll), self.ll_words, C.c_void_p(t.data_ptr()),
                                                 C.c_void_p(out.data_ptr()), t.numel(), DT[t.dtype], OPS[op],
                                                 self._stream(stream)), "all_reduce_ll")
        self.launches += n
        return out

    def barrier(self, channel: int = 2, stream=None):
        self.launches += self._chk(self.lib.bnet_barrier(self.h, channel, self._stream(stream)), "barrier")

    def fused_allreduce_sgd(self, grad: torch.Tensor, param: torch.Tensor, master: torch.Tensor, mom: torch.Tensor,
                            lr: float, momentum: float, weight_decay: float, grad_scale: float | None = None,
                            zero_grads: bool = True, channel: int = 0, nblocks: int = 0, stream=None,
                            hp: torch.Tensor | None = None):
        """One kernel: mean-reduce ``grad`` across ranks, SGD-update this rank's fp32 shard
        (``master``/``mom``: numel/world each) and write the new ``param`` on every rank.
        ``hp``: optional 4-element fp32 CUDA tensor {lr, momentum, weight_decay, grad_scale} that the kernel reads when
        it runs (overrides the scalar arguments) — lets a captured CUDA graph follow a learning-rate schedule."""
        gs = (1.0 / self.world) if grad_scale is None else grad_scale
        self._fused_step("fused_allreduce_sgd" if hp is None else "fused_allreduce_sgd_hp", grad, param, (master, mom),
                         (lr, momentum, weight_decay, gs), hp, 4, zero_grads, channel, nblocks, stream)

    def fused_allreduce_adamw(self, grad: torch.Tensor, param: torch.Tensor, master: torch.Tensor, exp_avg: torch.Tensor,
                              exp_avg_sq: torch.Tensor, hp: torch.Tensor, zero_grads: bool = True, channel: int = 0,
                              nblocks: int = 0, stream=None):
        """One kernel: sum-reduce ``grad`` across ranks, AdamW-update this rank's fp32 shard (``master`` / ``exp_avg`` /
        ``exp_avg_sq``: numel/world each) and write the new ``param`` on every rank.  ``hp``: fp32 CUDA tensor of 8
        elements {lr, beta1, beta2, eps, weight_decay, grad_scale, step, reserved} that the kernel reads when it runs;
        ``step`` counts the steps already taken and is not advanced here (the caller does that once per step)."""
        assert hp is not None
        self._fused_step("fused_allreduce_adamw", grad, param, (master, exp_avg, exp_avg_sq), (), hp, 8, zero_grads, channel,
                         nblocks, stream)

    def _fused_step(self, name, grad, param, state, scalars, hp, hp_words, zero_grads, channel, nblocks, stream):
        """Calls ``bnet_<name>``: the checks both fused optimizers share.  ``state``: the fp32 shards, master first;
        ``hp``: the device hyper-parameter block of at least ``hp_words`` floats, passed instead of ``scalars``."""
        assert grad.numel() == param.numel() and grad.dtype == param.dtype
        assert all(s.dtype == torch.float32 and s.numel() * self.world == grad.numel() for s in state)
        if hp is not None:
            assert hp.is_cuda and hp.dtype == torch.float32 and hp.numel() >= hp_words and hp.is_contiguous()
            scalars = (C.c_void_p(hp.data_ptr()),)
        n = self._chk(getattr(self.lib, "bnet_" + name)(
            self.h, self.offset_of(grad), self.offset_of(param), grad.numel(), DT[grad.dtype], *scalars,
            *(C.c_void_p(s.data_ptr()) for s in state), 1 if zero_grads else 0, channel, nblocks, self._stream(stream)), name)
        self.launches += n

    # ------------------------------------------------------------------ fused step with gradient clipping (three stages)
    def fused_clip_reduce_norm(self, grad: torch.Tensor, scratch: torch.Tensor, partial: torch.Tensor, channel: int = 0,
                               nblocks: int = 0, stream=None):
        """Stage 1, per bucket: sum-reduce ``grad`` across ranks into this rank's fp32 ``scratch`` shard (numel/world),
        write each CTA's sum of squares to its slot of the float64 ``partial`` row (``CLIP_ROW`` slots) and zero ``grad``."""
        assert scratch.dtype == torch.float32 and scratch.is_contiguous() and scratch.numel() * self.world == grad.numel()
        assert partial.is_cuda and partial.dtype == torch.float64 and partial.is_contiguous() and partial.numel() >= CLIP_ROW
        n = self._chk(self.lib.bnet_fused_clip_reduce_norm(
            self.h, self.offset_of(grad), grad.numel(), DT[grad.dtype], C.c_void_p(scratch.data_ptr()),
            C.c_void_p(partial.data_ptr()), channel, nblocks, self._stream(stream)), "fused_clip_reduce_norm")
        self.launches += n

    def fused_accum_reduce_norm(self, grad: torch.Tensor, scratch: torch.Tensor, partial: torch.Tensor, channel: int = 0,
                                nblocks: int = 0, stream=None):
        """Stage 1 of a micro-batch that accumulates (gradient accumulation): like ``fused_clip_reduce_norm``, but ADD the
        rank-summed ``grad`` to this rank's fp32 ``scratch`` shard (scratch + g, in fp32); ``partial`` gets the sums of
        squares of the new scratch values.  Zeroes ``grad``."""
        assert scratch.dtype == torch.float32 and scratch.is_contiguous() and scratch.numel() * self.world == grad.numel()
        assert partial.is_cuda and partial.dtype == torch.float64 and partial.is_contiguous() and partial.numel() >= CLIP_ROW
        n = self._chk(self.lib.bnet_fused_accum_reduce_norm(
            self.h, self.offset_of(grad), grad.numel(), DT[grad.dtype], C.c_void_p(scratch.data_ptr()),
            C.c_void_p(partial.data_ptr()), channel, nblocks, self._stream(stream)), "fused_accum_reduce_norm")
        self.launches += n

    def fused_clip_coef(self, partials: torch.Tensor, xchg: torch.Tensor, clip: torch.Tensor, grad_scale: float | None = None,
                        channel: int = 0, stream=None):
        """Stage 2, once per step: the global norm from every rank's ``partials`` ([buckets, CLIP_ROW] float64), exchanged
        through the heap tensor ``xchg`` (at least ``world`` float64), times ``grad_scale`` (default 1/world: the norm of
        the mean gradient); writes total_norm and clip_coef into ``clip`` ({max_norm, total_norm, clip_coef, reserved})."""
        assert partials.is_cuda and partials.dtype == torch.float64 and partials.is_contiguous()
        assert partials.dim() == 2 and partials.shape[1] == CLIP_ROW
        assert xchg.numel() * xchg.element_size() >= 8 * self.world
        assert clip.is_cuda and clip.dtype == torch.float32 and clip.numel() >= 4 and clip.is_contiguous()
        gs = (1.0 / self.world) if grad_scale is None else grad_scale
        n = self._chk(self.lib.bnet_fused_clip_coef(self.h, C.c_void_p(partials.data_ptr()), partials.shape[0],
                                                    self.offset_of(xchg), gs, C.c_void_p(clip.data_ptr()), channel,
                                                    self._stream(stream)), "fused_clip_coef")
        self.launches += n

    def fused_clip_apply_sgd(self, param: torch.Tensor, scratch: torch.Tensor, clip: torch.Tensor, master: torch.Tensor,
                             mom: torch.Tensor, lr: float, momentum: float, weight_decay: float, grad_scale: float | None = None,
                             channel: int = 0, nblocks: int = 0, stream=None, hp: torch.Tensor | None = None):
        """Stage 3, per bucket: the SGD step of ``fused_allreduce_sgd`` from ``scratch`` times clip_coef, and the new
        ``param`` on every rank."""
        gs = (1.0 / self.world) if grad_scale is None else grad_scale
        self._clip_apply("fused_clip_apply_sgd" if hp is None else "fused_clip_apply_sgd_hp", param, scratch, clip,
                         (master, mom), (lr, momentum, weight_decay, gs), hp, 4, channel, nblocks, stream)

    def fused_clip_apply_adamw(self, param: torch.Tensor, scratch: torch.Tensor, clip: torch.Tensor, master: torch.Tensor,
                               exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor, hp: torch.Tensor, channel: int = 0,
                               nblocks: int = 0, stream=None):
        """Stage 3, per bucket: the AdamW step of ``fused_allreduce_adamw`` from ``scratch`` times clip_coef, and the new
        ``param`` on every rank."""
        assert hp is not None
        self._clip_apply("fused_clip_apply_adamw", param, scratch, clip, (master, exp_avg, exp_avg_sq), (), hp, 8, channel,
                         nblocks, stream)

    def _clip_apply(self, name, param, scratch, clip, state, scalars, hp, hp_words, channel, nblocks, stream):
        assert scratch.dtype == torch.float32 and scratch.is_contiguous() and scratch.numel() * self.world == param.numel()
        assert clip.is_cuda and clip.dtype == torch.float32 and clip.numel() >= 4 and clip.is_contiguous()
        assert all(s.dtype == torch.float32 and s.numel() * self.world == param.numel() for s in state)
        if hp is not None:
            assert hp.is_cuda and hp.dtype == torch.float32 and hp.numel() >= hp_words and hp.is_contiguous()
            scalars = (C.c_void_p(hp.data_ptr()),)
        n = self._chk(getattr(self.lib, "bnet_" + name)(
            self.h, self.offset_of(param), param.numel(), DT[param.dtype], C.c_void_p(scratch.data_ptr()),
            C.c_void_p(clip.data_ptr()), *scalars, *(C.c_void_p(s.data_ptr()) for s in state), channel, nblocks,
            self._stream(stream)), name)
        self.launches += n

    # ------------------------------------------------------------------ LARS (staged step: norm, trust, apply)
    def lars_segments(self, table, shard_vecs: int, ntensors: int) -> torch.Tensor:
        """Validate a bucket's LARS segment table on the host (``check_lars_segments``) and upload it: the kernels
        accept only tables that went through here.  Returns the [nseg, 4] int32 device tensor."""
        nslots = check_lars_segments(table, shard_vecs, ntensors)
        t = torch.as_tensor(table, dtype=torch.int32).reshape(-1, 4).to(f"cuda:{self.device}").contiguous()
        self._lars_tables[t.data_ptr()] = ("seg", t, shard_vecs, nslots, ntensors)
        return t

    def lars_tensors(self, table, nslots: int) -> torch.Tensor:
        """Validate a LARS tensor table against `nslots` norm slots (``check_lars_tensors``) and upload it."""
        check_lars_tensors(table, nslots)
        t = torch.as_tensor(table, dtype=torch.int32).reshape(-1, 4).to(f"cuda:{self.device}").contiguous()
        self._lars_tables[t.data_ptr()] = ("tensor", t, nslots, t.shape[0], t.shape[0])
        return t

    def _lars_table(self, t, kind, size):
        rec = self._lars_tables.get(t.data_ptr())
        if rec is None or rec[0] != kind or rec[1] is not t or rec[2] != size:
            raise ValueError(f"LARS {kind} table was not validated for this shape: upload it with SymmComm.lars_{kind}s")
        return rec

    def fused_lars_norm(self, master: torch.Tensor, scratch: torch.Tensor, segs: torch.Tensor, slots: torch.Tensor,
                        dtype: torch.dtype, nblocks: int = 0, stream=None):
        """Per bucket, after stage 1: per chunk of each segment of ``segs`` (from ``lars_segments``), the float64 sums of
        squares of this rank's fp32 ``master`` and ``scratch`` shard into the rows {sum w^2, sum g^2} of ``slots``
        ([nslots, 2] float64).  ``dtype``: the parameters' dtype, which sets the elements per 16-byte vector."""
        assert dtype in (torch.float32, torch.bfloat16)
        assert master.is_cuda and master.dtype == torch.float32 and master.is_contiguous()
        assert scratch.is_cuda and scratch.dtype == torch.float32 and scratch.is_contiguous() and scratch.numel() == master.numel()
        per_vec = 16 // torch.empty((), dtype=dtype).element_size()
        assert master.numel() % per_vec == 0
        nslots = self._lars_table(segs, "seg", master.numel() // per_vec)[3]
        assert slots.is_cuda and slots.dtype == torch.float64 and slots.is_contiguous() and tuple(slots.shape) == (nslots, 2)
        n = self._chk(self.lib.bnet_fused_lars_norm(
            self.h, master.numel() * self.world, DT[dtype], C.c_void_p(master.data_ptr()), C.c_void_p(scratch.data_ptr()),
            C.c_void_p(segs.data_ptr()), segs.shape[0], C.c_void_p(slots.data_ptr()), nslots, nblocks, self._stream(stream)),
            "fused_lars_norm")
        self.launches += n

    def fused_lars_trust(self, slots: torch.Tensor, tensors: torch.Tensor, xchg: torch.Tensor, clip: torch.Tensor,
                         hp: torch.Tensor, scal: torch.Tensor, trust: torch.Tensor, channel: int = 0, stream=None):
        """Once per step, after every norm launch: per tensor of ``tensors`` (from ``lars_tensors``), the norms over all
        ranks (exchanged through the heap tensor ``xchg``, at least 2 * world * ntensors float64), the trust ratio into
        ``trust`` ([ntensors] fp32) and the update scalars {grad scale, weight decay} into ``scal`` ([ntensors, 2] fp32).
        ``clip``: the 4-float clip block (its clip_coef is used); ``hp``: the 8-float LARS block."""
        T = tensors.shape[0]
        self._lars_table(tensors, "tensor", slots.shape[0])
        assert slots.is_cuda and slots.dtype == torch.float64 and slots.is_contiguous() and slots.dim() == 2 and slots.shape[1] == 2
        assert xchg.numel() * xchg.element_size() >= 16 * self.world * T
        assert clip.is_cuda and clip.dtype == torch.float32 and clip.numel() >= 4 and clip.is_contiguous()
        assert hp.is_cuda and hp.dtype == torch.float32 and hp.numel() >= 8 and hp.is_contiguous()
        assert scal.is_cuda and scal.dtype == torch.float32 and scal.is_contiguous() and tuple(scal.shape) == (T, 2)
        assert trust.is_cuda and trust.dtype == torch.float32 and trust.is_contiguous() and trust.numel() == T
        n = self._chk(self.lib.bnet_fused_lars_trust(
            self.h, C.c_void_p(slots.data_ptr()), C.c_void_p(tensors.data_ptr()), T, self.offset_of(xchg),
            C.c_void_p(clip.data_ptr()), C.c_void_p(hp.data_ptr()), C.c_void_p(scal.data_ptr()), C.c_void_p(trust.data_ptr()),
            channel, self._stream(stream)), "fused_lars_trust")
        self.launches += n

    def fused_lars_apply(self, param: torch.Tensor, scratch: torch.Tensor, segs: torch.Tensor, scal: torch.Tensor,
                         hp: torch.Tensor, master: torch.Tensor, mom: torch.Tensor, channel: int = 0, nblocks: int = 0,
                         stream=None):
        """Per bucket, after the trust kernel: the SGD step of ``fused_clip_apply_sgd`` from ``scratch``, with each
        tensor's scalars from ``scal`` ([ntensors, 2], as many rows as the tensor count ``segs`` was validated for) and
        lr and momentum from ``hp``, and the new ``param`` on every rank."""
        assert scratch.dtype == torch.float32 and scratch.is_contiguous() and scratch.numel() * self.world == param.numel()
        assert all(s.dtype == torch.float32 and s.is_contiguous() and s.numel() * self.world == param.numel() for s in (master, mom))
        rec = self._lars_table(segs, "seg", param.numel() * param.element_size() // 16 // self.world)
        assert scal.is_cuda and scal.dtype == torch.float32 and scal.is_contiguous() and tuple(scal.shape) == (rec[4], 2)
        assert hp.is_cuda and hp.dtype == torch.float32 and hp.numel() >= 8 and hp.is_contiguous()
        n = self._chk(self.lib.bnet_fused_lars_apply(
            self.h, self.offset_of(param), param.numel(), DT[param.dtype], C.c_void_p(scratch.data_ptr()),
            C.c_void_p(segs.data_ptr()), segs.shape[0], C.c_void_p(scal.data_ptr()), C.c_void_p(hp.data_ptr()),
            C.c_void_p(master.data_ptr()), C.c_void_p(mom.data_ptr()), channel, nblocks, self._stream(stream)), "fused_lars_apply")
        self.launches += n

    # ------------------------------------------------------------------ parameter groups: per-group lr and weight decay
    def group_segments(self, table, shard_vecs: int, ngroups: int) -> torch.Tensor:
        """Validate a bucket's parameter-group segment table on the host (``check_group_segments``) and upload it: the
        grouped kernels accept only tables that went through here.  Returns the [nseg, 4] int32 device tensor."""
        check_group_segments(table, shard_vecs, ngroups)
        t = torch.as_tensor(table, dtype=torch.int32).reshape(-1, 4).to(f"cuda:{self.device}").contiguous()
        self._group_tables[t.data_ptr()] = (t, shard_vecs, ngroups)
        return t

    def _grouped_args(self, param, hp, hp_words, groups, segs):
        """The checks of the grouped entry points: ``hp`` the optimizer's device block, ``groups`` the [G, 4] fp32 group
        table (at least as many rows as ``segs`` was validated for), ``segs`` from ``group_segments`` for this shard."""
        rec = self._group_tables.get(segs.data_ptr())
        if rec is None or rec[0] is not segs or rec[1] != param.numel() * param.element_size() // 16 // self.world:
            raise ValueError("group segment table was not validated for this shard: upload it with SymmComm.group_segments")
        assert hp.is_cuda and hp.dtype == torch.float32 and hp.numel() >= hp_words and hp.is_contiguous()
        assert groups.is_cuda and groups.dtype == torch.float32 and groups.is_contiguous() and groups.dim() == 2
        assert groups.shape[1] == 4 and rec[2] <= groups.shape[0] <= GROUPS_MAX
        return (C.c_void_p(hp.data_ptr()), C.c_void_p(groups.data_ptr()), groups.shape[0], C.c_void_p(segs.data_ptr()),
                segs.shape[0])

    def fused_allreduce_sgd_groups(self, grad: torch.Tensor, param: torch.Tensor, master: torch.Tensor, mom: torch.Tensor,
                                   hp: torch.Tensor, groups: torch.Tensor, segs: torch.Tensor, zero_grads: bool = True,
                                   channel: int = 0, nblocks: int = 0, stream=None):
        """``fused_allreduce_sgd`` with every tensor's lr and weight decay from its group's row {lr, weight_decay,
        reserved, reserved} of ``groups``, found through ``segs``; momentum and gradient scale from the 4-float ``hp``."""
        self._fused_step("fused_allreduce_sgd_groups", grad, param, (master, mom), self._grouped_args(param, hp, 4, groups, segs),
                         None, 0, zero_grads, channel, nblocks, stream)

    def fused_allreduce_adamw_groups(self, grad: torch.Tensor, param: torch.Tensor, master: torch.Tensor,
                                     exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor, hp: torch.Tensor, groups: torch.Tensor,
                                     segs: torch.Tensor, zero_grads: bool = True, channel: int = 0, nblocks: int = 0,
                                     stream=None):
        """``fused_allreduce_adamw`` with every tensor's lr and weight decay from its group's row of ``groups``."""
        self._fused_step("fused_allreduce_adamw_groups", grad, param, (master, exp_avg, exp_avg_sq),
                         self._grouped_args(param, hp, 8, groups, segs), None, 0, zero_grads, channel, nblocks, stream)

    def fused_clip_apply_sgd_groups(self, param: torch.Tensor, scratch: torch.Tensor, clip: torch.Tensor, master: torch.Tensor,
                                    mom: torch.Tensor, hp: torch.Tensor, groups: torch.Tensor, segs: torch.Tensor,
                                    channel: int = 0, nblocks: int = 0, stream=None):
        """Stage 3, per bucket: ``fused_clip_apply_sgd`` with the per-group lr and weight decay of ``groups``."""
        self._clip_apply("fused_clip_apply_sgd_groups", param, scratch, clip, (master, mom),
                         self._grouped_args(param, hp, 4, groups, segs), None, 0, channel, nblocks, stream)

    def fused_clip_apply_adamw_groups(self, param: torch.Tensor, scratch: torch.Tensor, clip: torch.Tensor,
                                      master: torch.Tensor, exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor, hp: torch.Tensor,
                                      groups: torch.Tensor, segs: torch.Tensor, channel: int = 0, nblocks: int = 0,
                                      stream=None):
        """Stage 3, per bucket: ``fused_clip_apply_adamw`` with the per-group lr and weight decay of ``groups``."""
        self._clip_apply("fused_clip_apply_adamw_groups", param, scratch, clip, (master, exp_avg, exp_avg_sq),
                         self._grouped_args(param, hp, 8, groups, segs), None, 0, channel, nblocks, stream)

    # ------------------------------------------------------------------ exponential moving average of the master weights
    def ema_update(self, master: torch.Tensor, ema: torch.Tensor, blk: torch.Tensor, nblocks: int = 0, stream=None):
        """Per bucket, after the optimizer step's last update: on an EMA step of the 4-float device block ``blk``
        ({1 - decay, every, step, n_averaged}), ``ema`` becomes a copy of ``master`` (n_averaged == 0) or
        ``torch.lerp(ema, master, 1 - decay)``; on other steps neither is touched.  Both are this rank's fp32 shards."""
        assert master.is_cuda and master.dtype == torch.float32 and master.is_contiguous()
        assert ema.is_cuda and ema.dtype == torch.float32 and ema.is_contiguous() and ema.numel() == master.numel()
        assert blk.is_cuda and blk.dtype == torch.float32 and blk.numel() >= 4 and blk.is_contiguous()
        n = self._chk(self.lib.bnet_ema_update(self.h, master.numel(), C.c_void_p(master.data_ptr()),
                                               C.c_void_p(ema.data_ptr()), C.c_void_p(blk.data_ptr()), nblocks,
                                               self._stream(stream)), "ema_update")
        self.launches += n

    def ema_advance(self, blk: torch.Tensor, stream=None):
        """Once per optimizer step, after every bucket's ``ema_update``: count the step in ``blk``, and the EMA update
        when it was an EMA step."""
        assert blk.is_cuda and blk.dtype == torch.float32 and blk.numel() >= 4 and blk.is_contiguous()
        n = self._chk(self.lib.bnet_ema_advance(self.h, C.c_void_p(blk.data_ptr()), self._stream(stream)), "ema_advance")
        self.launches += n

    # ------------------------------------------------------------------ collectives on ordinary tensors
    # The kernels above work on heap tensors in place.  These wrappers accept any CUDA tensor: they stage it
    # through a heap buffer (allocated once, same offset on every rank — every rank must make the same calls)
    # and use the all-reduce kernels, the barrier kernel and peer mappings of the heap.
    def _stage(self, min_bytes: int = 0) -> torch.Tensor:
        if getattr(self, "_stage_buf", None) is None:
            free = self.heap_bytes - self._bump - (1 << 16)
            want = max(min(32 << 20, free), 0)
            if want < 16 * self.world:
                raise MemoryError("no room left in the symmetric heap for a staging buffer")
            self._stage_buf = self.alloc(want // (16 * self.world) * (16 * self.world), torch.uint8)
        return self._stage_buf

    def _chunks(self, flat: torch.Tensor):
        """(offset, count, heap view of `count` elements padded to the all-reduce quantum) over a flat tensor."""
        es = flat.element_size()
        q = 16 * self.world // es if es <= 16 else 1
        stage = self._stage().view(flat.dtype)
        cap = stage.numel() // q * q
        for off in range(0, flat.numel(), cap):
            m = min(cap, flat.numel() - off)
            yield off, m, stage[:(m + q - 1) // q * q]

    def all_reduce_tensor(self, t: torch.Tensor, op: str = "sum", algo: str = "auto", stream=None) -> torch.Tensor:
        """In-place all-reduce of any CUDA tensor (staged through the heap, chunked if larger than the stage)."""
        if self.world == 1:
            return t
        flat = t.reshape(-1) if t.is_contiguous() else t.contiguous().view(-1)
        with torch.cuda.stream(stream) if stream is not None else _null():
            for off, m, st in self._chunks(flat):
                st[:m].copy_(flat[off:off + m])
                if st.numel() > m:
                    st[m:].zero_()
                self.all_reduce(st, op, algo, stream=stream)
                flat[off:off + m].copy_(st[:m])
            if flat.data_ptr() != t.data_ptr():
                t.copy_(flat.view(t.shape))
        return t

    def broadcast_tensor(self, t: torch.Tensor, src: int = 0) -> torch.Tensor:
        """Every rank ends up with rank `src`'s values (read over NVLink from src's heap stage)."""
        if self.world == 1:
            return t
        flat = t.reshape(-1) if t.is_contiguous() else t.contiguous().view(-1)
        for off, m, st in self._chunks(flat):
            if self.rank == src:
                st[:m].copy_(flat[off:off + m])
            self.barrier()                       # src's stage is complete (and everybody is done with the last chunk)
            if self.rank != src:
                flat[off:off + m].copy_(self.peer_tensor(st[:m], src))
            self.barrier()                       # nobody still reads the stage
        if flat.data_ptr() != t.data_ptr():
            t.copy_(flat.view(t.shape))
        return t

    def all_gather_tensor(self, t: torch.Tensor) -> torch.Tensor:
        """Returns a [world, *t.shape] tensor with every rank's `t`."""
        out = torch.empty((self.world,) + tuple(t.shape), device=t.device, dtype=t.dtype)
        if self.world == 1:
            out[0].copy_(t)
            return out
        flat = t.reshape(-1) if t.is_contiguous() else t.contiguous().view(-1)
        of = out.view(self.world, -1)
        for off, m, st in self._chunks(flat):
            st[:m].copy_(flat[off:off + m])
            self.barrier()
            for p in range(self.world):
                of[p, off:off + m].copy_(st[:m] if p == self.rank else self.peer_tensor(st[:m], p))
            self.barrier()
        return out

    def reduce_scatter_tensor(self, t: torch.Tensor, op: str = "sum") -> torch.Tensor:
        """Returns this rank's 1/world slice of the element-wise reduction of every rank's `t` (numel % world == 0):
        each rank pulls only its own slice from every peer and accumulates in fp32."""
        if t.numel() % self.world:
            raise ValueError("reduce_scatter_tensor: numel must be a multiple of the world size")
        if op not in ("sum", "avg"):
            raise ValueError("reduce_scatter_tensor supports sum / avg")
        flat = t.reshape(-1) if t.is_contiguous() else t.contiguous().view(-1)
        n = flat.numel() // self.world
        if self.world == 1:
            return flat.clone()
        acc = torch.zeros(n, device=t.device, dtype=torch.float32)
        stage = self._stage().view(flat.dtype)
        cap = stage.numel()
        for off in range(0, n, cap // self.world):
            m = min(cap // self.world, n - off)
            # stage layout: world slices of m elements, slice p = what rank p will pull
            for p in range(self.world):
                stage[p * m:(p + 1) * m].copy_(flat[p * n + off:p * n + off + m])
            self.barrier()
            for p in range(self.world):
                src = stage if p == self.rank else self.peer_tensor(stage[:self.world * m], p)
                acc[off:off + m] += src[self.rank * m:(self.rank + 1) * m].float()
            self.barrier()
        if op == "avg":
            acc /= self.world
        return acc.to(t.dtype)


class _null:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


def init_process_group_from_env(backend: str | None = None):
    """torch.distributed bootstrap for one-process-per-GPU launches (torchrun env)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1 or dist.is_initialized():
        return
    local = int(os.environ.get("LOCAL_RANK", os.environ.get("RANK", "0")))
    if torch.cuda.is_available():
        torch.cuda.set_device(local)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29511")
    dist.init_process_group(backend or ("nccl" if torch.cuda.is_available() else "gloo"))

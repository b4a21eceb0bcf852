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
        assert out.is_contiguous() and out.numel() == t.numel() and out.dtype == t.dtype
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
        assert grad.numel() == param.numel() and grad.dtype == param.dtype
        assert master.dtype == torch.float32 and mom.dtype == torch.float32
        assert master.numel() * self.world == grad.numel() == mom.numel() * self.world
        if hp is not None:
            assert hp.is_cuda and hp.dtype == torch.float32 and hp.numel() >= 4 and hp.is_contiguous()
            n = self._chk(self.lib.bnet_fused_allreduce_sgd_hp(
                self.h, self.offset_of(grad), self.offset_of(param), grad.numel(), DT[grad.dtype], C.c_void_p(hp.data_ptr()),
                C.c_void_p(master.data_ptr()), C.c_void_p(mom.data_ptr()), 1 if zero_grads else 0, channel, nblocks,
                self._stream(stream)), "fused_allreduce_sgd_hp")
            self.launches += n
            return
        gs = (1.0 / self.world) if grad_scale is None else grad_scale
        n = self._chk(self.lib.bnet_fused_allreduce_sgd(
            self.h, self.offset_of(grad), self.offset_of(param), grad.numel(), DT[grad.dtype], lr, momentum,
            weight_decay, gs, C.c_void_p(master.data_ptr()), C.c_void_p(mom.data_ptr()), 1 if zero_grads else 0,
            channel, nblocks, self._stream(stream)), "fused_allreduce_sgd")
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

"""Data-parallel training engine on top of the fused bnet kernels.

The reference accelerates PyTorch/Bagua DDP by moving NCCL's all-reduce traffic faster
(reference README.md:52-84).  Here the data-parallel step itself is re-designed for an
NVSwitch box:

* parameters and gradients live in flat buffers inside the symmetric heap; ``p.data`` is a view, and every
  gradient has a slice of the flat gradient buffer that its producer writes directly (``ops/grad_target.py``) or
  that a hook copies it into — autograd never accumulates (no add pass, no bucket copy-in/copy-out);
* when the last gradient of a bucket has been produced, ONE kernel on a side stream
  reduces the bucket in the switch (NVLS), applies SGD+momentum+weight-decay on the owning
  rank's fp32 master shard, writes the new bf16 parameters to every rank and re-zeroes the
  gradients — overlapping the rest of the backward pass;
* optimizer state is sharded 1/world (ZeRO-1 style) for free.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from .comm import SymmComm


def plan_buckets(numels, element_size: int, world: int, bucket_mb: float):
    """Lay parameters out in the flat heap buffers.  Returns ([(start, numel, [(param index, offset), ...]), ...], total).

    * gradients become ready roughly in reverse registration order, so buckets are filled in that order;
    * every tensor starts on a 16-byte boundary (8 elements) inside the flat buffer;
    * every bucket is a whole number of 16-byte vectors per rank (`quantum`), so the fused kernel can shard it 1/world;
    * a bucket closes when the next tensor would push it past `bucket_mb`."""
    quantum = 16 * world // element_size * 8
    cap = int(bucket_mb * (1 << 20)) // element_size
    plan = []
    start, numel, members = 0, 0, []
    offset = 0
    for pi in reversed(range(len(numels))):
        n = numels[pi]
        if members and numel + n > cap:
            numel = (numel + quantum - 1) // quantum * quantum
            offset += numel
            plan.append((start, numel, members))
            start, numel, members = offset, 0, []
        members.append((pi, start + numel))
        numel += (n + 7) // 8 * 8
    numel = (numel + quantum - 1) // quantum * quantum
    offset += numel
    plan.append((start, numel, members))
    return plan, offset


def direct_grads_self_check(device=None, group=None, steps: int = 3, make_model=None, make_comm=None, make_batch=None,
                            use_graph: bool = True, fused: bool = True, verbose: bool = False):
    """Do adopted gradients (``BNET_DIRECT_GRADS=1``: producers write into the flat buffer, ``p.grad`` stays ``None``) train like
    accumulated ones (``BNET_DIRECT_GRADS=0``: autograd adds into views of the flat buffer) on THIS machine?

    Two engines are built from the same seed on a small full-width VGG16 (64-multiple channels, so the wgmma producers that
    write in place take part; 32 x 32 images), both run `steps` steps — captured in a CUDA graph like the benchmark's — and the
    fp32 master-weight UPDATES are compared (relative L2 error, over all of them and per parameter tensor: an update is what a
    misplaced or missing gradient changes, and the classifier's updates can outweigh a whole family of lost ones in the total).
    `group`: a single-rank process group when the job has more ranks (nothing here may wait for a peer).
    Returns (verdict, detail).  Any exception is a failed check, not an error: the caller falls back to accumulation."""
    import gc
    import os

    saved = os.environ.get("BNET_DIRECT_GRADS")
    detail = {}
    try:
        updates, losses, segments = {}, {}, []
        for mode in ("0", "1"):
            os.environ["BNET_DIRECT_GRADS"] = mode
            torch.manual_seed(4321)
            if make_model is not None:
                model = make_model()
            else:
                from ..models import build_model

                model = build_model("vgg16", fc_dim=256, image_size=32, num_classes=16, dropout=0.0, **({"fused": True} if fused else {}))
                model = model.to(device).to(torch.bfloat16).to(memory_format=torch.channels_last)
            model.train()
            if make_batch is not None:
                x, y = make_batch()
            else:
                x = torch.randn(8, 3, 32, 32, device=device, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
                y = torch.randint(0, 16, (8,), device=device)
            eng = BnetDDP(model, lr=0.05, momentum=0.9, weight_decay=1e-4, bucket_mb=8.0, group=group,
                          comm=make_comm() if make_comm is not None else None, extra_heap_bytes=8 << 20)
            assert eng._direct_grads == (mode == "1")
            before = torch.cat([b.master.reshape(-1).clone() for b in eng.buckets])
            if use_graph:
                eng.enable_cuda_graph(True)
            loss = None
            for _ in range(steps):
                loss = eng.train_step(x, y)
            if x.is_cuda:
                torch.cuda.synchronize()
            after = torch.cat([b.master.reshape(-1) for b in eng.buckets])
            updates[mode] = (after - before).double()
            if sum(b.master.numel() for b in eng.buckets) == eng.flat_param.numel():
                # every master covers its whole bucket (one rank): where each parameter's update sits in `after`
                base, es, pos, segments = eng.flat_param.data_ptr(), eng.flat_param.element_size(), 0, []
                for b in eng.buckets:
                    segments += [(pos + (p.data_ptr() - base) // es - b.start, p.numel()) for p in b.params]
                    pos += b.master.numel()
            losses[mode] = float(loss)
            detail[f"grad_copies_{'adopt' if mode == '1' else 'accumulate'}"] = int(eng.grad_copies)
            for h in eng._hooks:
                h.remove()
            del eng, model, before, after
            gc.collect()
        ref, got = updates["0"], updates["1"]
        finite = bool(torch.isfinite(got).all()) and bool(torch.isfinite(ref).all())
        err = float((got - ref).norm() / ref.norm().clamp_min(1e-30)) if finite else float("inf")
        worst = 0.0
        if finite and segments:
            for s, n in segments:
                d, r = float((got[s:s + n] - ref[s:s + n]).norm()), float(ref[s:s + n].norm())
                worst = max(worst, d / r if r > 0 else (0.0 if d == 0 else float("inf")))
        detail.update({"rel_l2_error_of_updates": err, "max_rel_l2_error_per_tensor": worst, "loss_accumulate": losses["0"],
                       "loss_adopt": losses["1"]})
        ok = (finite and float(ref.norm()) > 0 and err < 0.05 and worst < 0.05
              and abs(losses["0"] - losses["1"]) <= 0.05 * max(1.0, abs(losses["0"])))
    except Exception as ex:   # noqa: BLE001 - a failed check, whatever the reason
        ok = False
        detail["error"] = f"{type(ex).__name__}: {str(ex)[:200]}"
    finally:
        if saved is None:
            os.environ.pop("BNET_DIRECT_GRADS", None)
        else:
            os.environ["BNET_DIRECT_GRADS"] = saved
    if verbose:
        print(f"direct_grads_self_check: {ok} {detail}")
    return ok, detail


class _Bucket:
    __slots__ = ("params", "start", "numel", "ready", "grad", "param", "master", "mom")

    def __init__(self):
        self.params = []
        self.start = 0
        self.numel = 0
        self.ready = 0


class BnetDDP(torch.nn.Module):
    """Wraps ``module``; owns the optimizer (SGD with momentum, fused into the collective).

    bucket_mb sizes buckets for launch latency and overlap (NVSwitch: no per-link bound).
    """

    def __init__(self, module: torch.nn.Module, lr: float = 0.01, momentum: float = 0.9, weight_decay: float = 0.0,
                 bucket_mb: float = 64.0, comm: SymmComm | None = None, extra_heap_bytes: int = 64 << 20,
                 nblocks: int = 0, group=None):
        super().__init__()
        self.module = module
        self.lr, self.momentum, self.weight_decay = lr, momentum, weight_decay
        self.nblocks = nblocks
        params = [p for p in module.parameters() if p.requires_grad]
        if not params:
            raise ValueError("module has no trainable parameters")
        dtype = params[0].dtype
        if any(p.dtype != dtype for p in params):
            raise ValueError("BnetDDP expects a single parameter dtype (bf16 or fp32)")
        if dtype not in (torch.bfloat16, torch.float32):
            raise ValueError(f"unsupported parameter dtype {dtype}")
        self.dtype = dtype
        es = params[0].element_size()
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        plan, total = plan_buckets([p.numel() for p in params], es, world, bucket_mb)
        self.buckets: list[_Bucket] = []
        layout = []
        for start, numel, members in plan:
            b = _Bucket()
            b.start, b.numel = start, numel
            for pi, off in members:
                b.params.append(params[pi])
                layout.append((params[pi], b, off))
            self.buckets.append(b)

        dev = params[0].device
        if dev.type == "cuda" and any(p.dim() == 4 and p.dtype == torch.bfloat16 for p in params):
            # once-per-process kernel verdicts (a child-process self-check the first time on a machine) are settled here,
            # before the heap's rendezvous lines the ranks up again and long before the first cross-rank kernel barrier
            from ..ops import tc_conv

            try:
                tc_conv.prepare()
            except Exception:   # noqa: BLE001 - an unsettled verdict only means the library kernels are used
                pass
        if comm is None:
            comm = SymmComm(2 * total * es + extra_heap_bytes + (1 << 20), device=dev.index, group=group)
        self.comm = comm
        self.flat_param = comm.alloc(total, dtype)
        self.flat_grad = comm.alloc(total, dtype)
        self.flat_param.zero_()
        self.flat_grad.zero_()
        def shaped(flat, off, p):
            # keep a channels_last parameter channels_last inside the flat buffer (cuDNN's
            # preferred filter layout on tensor cores): same bytes, permuted view
            seg = flat[off:off + p.numel()]
            if p.dim() == 4 and not p.is_contiguous() and p.is_contiguous(memory_format=torch.channels_last):
                n, c, h, w = p.shape
                return seg.view(n, h, w, c).permute(0, 3, 1, 2)
            return seg.view(p.shape)

        # Gradients: every parameter owns a slice of the flat gradient buffer the fused kernels read.  p.grad stays None
        # between steps, so autograd ADOPTS what a backward function hands it instead of adding it into an existing
        # tensor (an add is three passes over the parameter's bytes; with 138 M parameters that was 32 kernels and 5 % of
        # a VGG16 step).  Producers that can write anywhere look the slice up (ops/grad_target.py) and write straight
        # into it; whatever arrives in a tensor of its own is copied there by the hook below.
        # BNET_DIRECT_GRADS=0 brings the accumulate-into-a-view behaviour back (p.grad = the slice, autograd adds into it).
        import os

        from ..ops import grad_target

        self._direct_grads = os.environ.get("BNET_DIRECT_GRADS", "1") != "0"
        self._release = grad_target.release
        self._grad_view: dict[int, torch.Tensor] = {}
        with torch.no_grad():
            for p, b, off in layout:
                view = shaped(self.flat_param, off, p)
                view.copy_(p.data)
                p.data = view
                gview = shaped(self.flat_grad, off, p)
                self._grad_view[id(p)] = gview
                if self._direct_grads:
                    grad_target.register(p, gview, owner=self)
                    p.grad = None
                else:
                    p.grad = gview
        self._param_bucket = {id(p): b for p, b, _ in layout}
        # identical start on every rank (like DDP's initial broadcast): rank 0 wins, through our own all-reduce
        if comm.world > 1:
            if comm.rank != 0:
                self.flat_param.zero_()
            torch.cuda.synchronize()
            dist.barrier(group=group)
            comm.all_reduce(self.flat_param, "sum")
            torch.cuda.synchronize()
        # fp32 master weights + momentum for this rank's shard of every bucket
        for b in self.buckets:
            b.grad = self.flat_grad[b.start:b.start + b.numel]
            b.param = self.flat_param[b.start:b.start + b.numel]
            shard = b.numel // comm.world
            b.master = b.param[comm.rank * shard:(comm.rank + 1) * shard].float().contiguous()
            b.mom = torch.zeros_like(b.master)
        self.comm_stream = torch.cuda.Stream(device=dev, priority=-1)
        self.grad_copies = 0             # gradients that had to be copied into their slice (not written there by their producer)
        self._hooks = [p.register_post_accumulate_grad_hook(self._on_grad) for p in params]
        self._inflight = False
        torch.cuda.synchronize()
        if comm.world > 1:
            dist.barrier(group=group)

    # ------------------------------------------------------------------ autograd integration
    def _on_grad(self, p: torch.Tensor):
        g = p.grad
        if g is not None and self._direct_grads:
            view = self._grad_view[id(p)]
            if g.data_ptr() != view.data_ptr() or g.stride() != view.stride():
                view.copy_(g)                     # produced in a tensor of its own: put it where the fused kernel reads
                self.grad_copies += 1
            p.grad = None                         # (the slice is zeroed by the fused kernel; the next backward adopts again)
            self._release(p)                      # its slice may be handed to a producer again (ops/grad_target.py)
        b = self._param_bucket[id(p)]
        b.ready += 1
        if b.ready == len(b.params):
            self._launch(b)

    def _launch(self, b: _Bucket):
        cur = torch.cuda.current_stream()
        ev = torch.cuda.Event()
        ev.record(cur)
        self.comm_stream.wait_event(ev)          # the bucket's gradients are complete on the compute stream
        self.comm.fused_allreduce_sgd(b.grad, b.param, b.master, b.mom, self.lr, self.momentum, self.weight_decay,
                                      zero_grads=True, channel=0, nblocks=self.nblocks, stream=self.comm_stream,
                                      hp=getattr(self, "_hp", None))
        b.ready = 0
        self._inflight = True

    def finish_step(self):
        """Make the updated parameters visible to the compute stream (call after backward)."""
        for b in self.buckets:
            if b.ready:                           # parameters that got no gradient this step
                self._launch(b)
        if self._inflight:
            torch.cuda.current_stream().wait_stream(self.comm_stream)
            self._inflight = False

    # ------------------------------------------------------------------ user API
    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def _eager_step(self, inputs, targets, loss_fn):
        out = self.module(inputs)
        loss = loss_fn(out.float(), targets)
        loss.backward()
        self.finish_step()
        return loss.detach()

    def enable_cuda_graph(self, enabled: bool = True):
        """Capture forward + backward + the fused collective/optimizer kernels (both streams) into ONE
        CUDA graph and replay it every step: the ~150 launches of a step cost one cudaGraphLaunch.
        Needs static shapes; re-captured when shapes or the learning rate change.  Every rank must
        make the same choice."""
        self._use_graph = enabled
        self._graph = None

    def _capture(self, inputs, targets, loss_fn, key):
        from ..ops import fused_nn

        cur = torch.cuda.current_stream()
        self._gx = inputs.clone(memory_format=torch.preserve_format)
        self._gy = targets.clone()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):               # warm-up on a side stream (cuDNN autotune, allocator)
            # The warm-up runs REAL steps (the fused optimizer included: every rank has to take part in its
            # barriers), so everything a step mutates is saved first and put back afterwards — parameters, fp32
            # master weights, momentum, module buffers (BatchNorm running statistics).  A (re)capture therefore
            # leaves the training trajectory exactly where eager mode would have it; checkpoint/resume stays
            # step-exact.
            saved = [self.flat_param.clone()] + [t.clone() for b in self.buckets for t in (b.master, b.mom)]
            bufs = [t for t in self.module.buffers() if t.is_cuda and t.numel()]
            saved_bufs = [t.clone() for t in bufs]
            for _ in range(2):
                self._eager_step(self._gx, self._gy, loss_fn)
            torch.cuda.current_stream().synchronize()
            if self.comm.world > 1:
                dist.barrier()                      # nobody restores while a peer's kernel still writes parameters
            it = iter(saved)
            self.flat_param.copy_(next(it))
            for b in self.buckets:
                b.master.copy_(next(it))
                b.mom.copy_(next(it))
            for t, s in zip(bufs, saved_bufs):
                t.copy_(s)
            del saved, saved_bufs
        cur.wait_stream(side)
        torch.cuda.synchronize()
        if self.comm.world > 1:
            dist.barrier()
        from ..ops import tc_linear

        l0, f0, t0 = self.comm.launches, fused_nn.LAUNCHES, tc_linear.LAUNCHES
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._gloss = self._eager_step(self._gx, self._gy, loss_fn)
        self._graph_launches = (self.comm.launches - l0, fused_nn.LAUNCHES - f0, tc_linear.LAUNCHES - t0)
        self._graph, self._graph_key = g, key
        torch.cuda.synchronize()
        if self.comm.world > 1:
            dist.barrier()

    def train_step(self, inputs: torch.Tensor, targets: torch.Tensor, loss_fn=None) -> torch.Tensor:
        """forward + backward + fused all-reduce/optimizer.  Returns the (device) loss tensor."""
        loss_fn = loss_fn or torch.nn.functional.cross_entropy
        if not getattr(self, "_use_graph", False):
            return self._eager_step(inputs, targets, loss_fn)
        from ..ops import fused_nn

        # with the hyper-parameters in device memory (after the first set_lr) the captured step does not depend on them
        hpkey = "device" if getattr(self, "_hp", None) is not None else (self.lr, self.momentum, self.weight_decay)
        # (a lambda written inline is a new function object every call, but always the same code object)
        fn_key = (getattr(loss_fn, "__code__", loss_fn), getattr(loss_fn, "__closure__", None) is None or id(loss_fn))
        key = (tuple(inputs.shape), inputs.dtype, tuple(targets.shape), targets.dtype, fn_key, hpkey)
        if self._graph is None or self._graph_key != key:
            self._capture(inputs, targets, loss_fn, key)
        self._gx.copy_(inputs, non_blocking=True)
        self._gy.copy_(targets, non_blocking=True)
        self._graph.replay()
        self.comm.launches += self._graph_launches[0]      # the replay re-issues every captured kernel of ours
        fused_nn.LAUNCHES += self._graph_launches[1]
        if self._graph_launches[2]:
            from ..ops import tc_linear

            tc_linear.LAUNCHES += self._graph_launches[2]  # (wgmma linear / convolution kernels captured in the step)
        return self._gloss

    def train_step_from_host(self, inputs_pinned: torch.Tensor, targets_pinned: torch.Tensor, loss_fn=None) -> float:
        """End-to-end step as a user runs it: H2D copy of this step's batch from pinned host
        memory, train_step, D2H read of the loss."""
        dev = self.flat_param.device
        x = inputs_pinned.to(dev, non_blocking=True)
        y = targets_pinned.to(dev, non_blocking=True)
        if x.dim() == 4:
            x = x.contiguous(memory_format=torch.channels_last)
        return float(self.train_step(x, y, loss_fn).item())

    def train_from_host(self, batches, loss_fn=None, lag: int = 1):
        """Training loop over an iterable of (inputs_pinned, targets_pinned) batches — the loader-facing API.
        Yields the loss of every step as a float, in order (one device→host read per step).

        * The host→device copy of batch i+1 is issued on a dedicated copy stream right after step i has been
          enqueued, so the PCIe transfer rides under step i's kernels instead of in front of step i+1 (what a
          DataLoader prefetcher with pin_memory does for eager PyTorch).
        * The loss of step i is copied to pinned memory asynchronously and handed out `lag` steps later (default 1),
          i.e. after step i+1 has been enqueued: the GPU never waits for the host to read a number.  `lag=0` reads
          each loss before the next step is launched."""
        dev = self.flat_param.device
        if getattr(self, "_h2d_stream", None) is None:
            self._h2d_stream = torch.cuda.Stream(device=dev)
        copy = self._h2d_stream
        lag = max(int(lag), 0)
        if len(getattr(self, "_loss_host", ())) < lag + 2:
            self._loss_host = [torch.zeros(1, dtype=torch.float32).pin_memory() for _ in range(lag + 2)]
        bufs = self._loss_host

        def stage(batch):
            xh, yh = batch
            with torch.cuda.stream(copy):
                x = xh.to(dev, non_blocking=True)
                y = yh.to(dev, non_blocking=True)
                if x.dim() == 4:
                    x = x.contiguous(memory_format=torch.channels_last)
                ev = torch.cuda.Event()
                ev.record(copy)
            return x, y, ev

        it = iter(batches)
        try:
            nxt = stage(next(it))
        except StopIteration:
            return
        pending = []                    # (event, pinned buffer) of steps whose loss has not been handed out yet
        step = 0
        while nxt is not None:
            x, y, ev = nxt
            cur = torch.cuda.current_stream()
            cur.wait_event(ev)
            x.record_stream(cur)        # allocated on the copy stream, consumed on the compute stream
            y.record_stream(cur)
            loss = self.train_step(x, y, loss_fn)
            hb = bufs[step % len(bufs)]
            step += 1
            hb.copy_(loss.detach().reshape(1).float(), non_blocking=True)   # this step's loss, D2H, asynchronous
            done = torch.cuda.Event()
            done.record(cur)
            pending.append((done, hb))
            try:
                nxt = stage(next(it))   # overlaps the step that was just enqueued
            except StopIteration:
                nxt = None
            while len(pending) > lag:
                e, b = pending.pop(0)
                e.synchronize()
                yield float(b[0])
        for e, b in pending:
            e.synchronize()
            yield float(b[0])

    # ------------------------------------------------------------------ checkpoint / resume
    # Model weights live in ordinary nn.Module tensors (views into the flat heap), so module.state_dict() /
    # load_state_dict() work unchanged.  The optimizer state is this rank's 1/world shard of the fp32 master
    # weights and momentum of every bucket.
    def optimizer_state_dict(self) -> dict:
        return {"lr": self.lr, "momentum": self.momentum, "weight_decay": self.weight_decay,
                "world": self.comm.world, "rank": self.comm.rank,
                "buckets": [{"master": b.master.detach().cpu(), "momentum": b.mom.detach().cpu()} for b in self.buckets]}

    def load_optimizer_state_dict(self, state: dict) -> None:
        if state["world"] != self.comm.world or state["rank"] != self.comm.rank or len(state["buckets"]) != len(self.buckets):
            raise ValueError("optimizer state was saved for a different world size / rank / bucket layout")
        for b, s in zip(self.buckets, state["buckets"]):
            if s["master"].shape != b.master.shape:
                raise ValueError("optimizer state shard does not match this bucket")
            b.master.copy_(s["master"])
            b.mom.copy_(s["momentum"])
        self.lr, self.momentum, self.weight_decay = state["lr"], state["momentum"], state["weight_decay"]
        if getattr(self, "_hp", None) is not None:
            self.set_lr(self.lr)              # hyper-parameters live in device memory: refresh them
        else:
            self._graph = None                # hyper-parameters are baked into a captured step

    def sync_master_from_params(self) -> None:
        """After module.load_state_dict(): rebuild the fp32 master shards from the (just loaded) parameters."""
        for b in self.buckets:
            shard = b.numel // self.comm.world
            b.master.copy_(b.param[self.comm.rank * shard:(self.comm.rank + 1) * shard].float())

    def broadcast_buffers(self, src: int = 0) -> None:
        """Copy rank `src`'s module buffers (BatchNorm running statistics, ...) to every rank — what torch DDP does
        before each forward with broadcast_buffers=True.  Call it before evaluation / checkpointing; training itself
        does not depend on it (batch statistics are local, like in DDP)."""
        if self.comm.world == 1:
            return
        for b in self.module.buffers():
            if b.is_cuda and b.numel():
                self.comm.broadcast_tensor(b, src=src)

    def set_lr(self, lr: float, momentum: float | None = None, weight_decay: float | None = None):
        """Learning-rate schedule hook.  From the first call on, the fused optimizer kernels read {lr, momentum,
        weight decay, 1/world} from a 4-float device tensor instead of baked-in launch arguments, so a captured CUDA
        graph is re-captured once (here) and then follows the schedule with one tiny host→device write per change."""
        self.lr = float(lr)
        if momentum is not None:
            self.momentum = float(momentum)
        if weight_decay is not None:
            self.weight_decay = float(weight_decay)
        vals = [self.lr, self.momentum, self.weight_decay, 1.0 / self.comm.world]
        if getattr(self, "_hp", None) is None:
            self._hp = torch.tensor(vals, dtype=torch.float32, device=self.flat_param.device)
            self._graph = None
        else:
            self._hp.copy_(torch.tensor(vals, dtype=torch.float32), non_blocking=False)

    @property
    def kernel_launches(self) -> int:
        return self.comm.launches

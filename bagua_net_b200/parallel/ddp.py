"""Data-parallel training engine on top of the fused bnet kernels.

The reference accelerates PyTorch/Bagua DDP by moving NCCL's all-reduce traffic faster
(reference README.md:52-84).  Here the data-parallel step itself is re-designed for an
NVSwitch box:

* parameters and gradients live in flat buffers inside the symmetric heap; ``p.data`` is a view, and every
  gradient has a slice of the flat gradient buffer that its producer writes directly (``ops/grad_target.py``) or
  that a hook copies it into — autograd never accumulates (no add pass, no bucket copy-in/copy-out);
* when the last gradient of a bucket has been produced, ONE kernel on a side stream
  reduces the bucket in the switch (NVLS), applies the optimizer (SGD+momentum+weight-decay, or AdamW) on the owning
  rank's fp32 master shard, writes the new bf16 parameters to every rank and re-zeroes the
  gradients — overlapping the rest of the backward pass;
* optimizer state is sharded 1/world (ZeRO-1 style) for free.
"""
from __future__ import annotations

import contextlib
import math

import torch
import torch.distributed as dist

from .comm import GROUPS_MAX, LARS_CHUNK, SymmComm


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


# The fp32 tensors the fused kernel updates in every bucket's shard, master weights first; also their state-dict keys.
_STATE_NAMES = {"sgd": ("master", "momentum"), "adamw": ("master", "exp_avg", "exp_avg_sq"), "lars": ("master", "momentum")}


def lars_segments(members, numels, start: int, numel: int, element_size: int, world: int, rank: int):
    """The LARS segment table of one bucket on one rank: rows [vec0, nvec, tensor, slot0] (include/bnet/bnet_coll.h).

    `members`: the bucket's [(parameter index, element offset in the flat buffer), ...] in offset order (plan_buckets);
    `numels`: every parameter's element count; `start` / `numel`: the bucket's element range.  A segment is the part
    of one tensor in this rank's shard, in 16-byte vectors relative to the shard.  Tensors start on 16-byte boundaries,
    so no vector holds two tensors; the zero padding after a tensor joins the segment before it (padding at the start of
    a shard joins the first segment, and a shard of padding alone becomes one segment of the bucket's last tensor).  The
    rows cover the shard exactly once, and slot0 counts the LARS_CHUNK-vector chunks of the segments before."""
    per_vec = 16 // element_size
    shard = numel // world // per_vec                     # vectors in every rank's shard
    lo = start + rank * shard * per_vec                   # the shard's element range
    hi = lo + shard * per_vec
    rows = []
    for pi, off in members:
        a, b = max(off, lo), min(off + numels[pi], hi)
        if a < b:
            rows.append([(a - lo) // per_vec, (b - lo + per_vec - 1) // per_vec, pi])
    if not rows:
        rows = [[0, shard, members[-1][0]]]
    rows[0][0] = 0
    for r, nxt in zip(rows, rows[1:]):
        r[1] = nxt[0]                                     # [first, end) -> padding joins the segment before
    rows[-1][1] = shard
    table, slot = [], 0
    for first, end, pi in rows:
        table.append([first, end - first, pi, slot])
        slot += (end - first + LARS_CHUNK - 1) // LARS_CHUNK
    return table


def group_segments(members, numels, group_of, start: int, numel: int, element_size: int, world: int, rank: int):
    """The parameter-group segment table of one bucket on one rank: rows [vec0, nvec, group, 0] (include/bnet/bnet_coll.h),
    the LARS segments of ``lars_segments`` with every tensor mapped to its group (``group_of[parameter index]``) and
    adjacent rows of the same group merged.  Padding goes with the segment it joins there."""
    rows = []
    for vec0, nvec, pi, _ in lars_segments(members, numels, start, numel, element_size, world, rank):
        if rows and rows[-1][2] == group_of[pi]:
            rows[-1][1] += nvec
        else:
            rows.append([vec0, nvec, group_of[pi], 0])
    return rows


# ------------------------------------------------------------------ the shard <-> full mapping of the optimizer state
def shard_pieces(plan, numels, world: int, rank: int) -> list:
    """Where every bucket's shard on one rank comes from: per bucket of ``plan`` (plan_buckets), the pieces
    ``(parameter index, first element in the parameter, count, offset in the shard)`` in shard order.  Elements are
    counted in the parameter's memory order (as the flat buffer holds it: ``memory_flat``).  Shard elements that no piece
    covers are padding (the 16-byte alignment after a tensor, the bucket quantum at its end), and a shard may hold no
    piece at all."""
    out = []
    for start, numel, members in plan:
        shard = numel // world
        lo, hi = start + rank * shard, start + (rank + 1) * shard
        pieces = []
        for pi, off in members:
            a, b = max(off, lo), min(off + numels[pi], hi)
            if a < b:
                pieces.append((pi, a - off, b - a, a - lo))
        out.append(pieces)
    return out


def shard_from_full(flats, pieces, shard: torch.Tensor) -> torch.Tensor:
    """Fill one bucket's ``shard`` from ``flats`` (every parameter's values, flat in memory order) along ``pieces`` (one
    bucket's entry of ``shard_pieces``); the padding becomes zero.  Returns ``shard``."""
    shard.zero_()
    for pi, p0, n, s0 in pieces:
        shard[s0:s0 + n].copy_(flats[pi][p0:p0 + n])
    return shard


def full_from_shard(flats, pieces, shard: torch.Tensor) -> None:
    """The inverse of ``shard_from_full``: copy the pieces of one bucket's ``shard`` into ``flats``; padding is dropped."""
    for pi, p0, n, s0 in pieces:
        flats[pi][p0:p0 + n].copy_(shard[s0:s0 + n])


def memory_flat(t: torch.Tensor) -> torch.Tensor:
    """A 1-D view of ``t`` in the element order the flat buffers use for a parameter of its layout: NHWC for a
    channels_last 4-D tensor (as BnetDDP keeps such filters), the logical order for a contiguous one."""
    if t.dim() == 4 and not t.is_contiguous() and t.is_contiguous(memory_format=torch.channels_last):
        return t.permute(0, 2, 3, 1).view(-1)
    return t.view(-1)


def no_weight_decay_groups(module: torch.nn.Module, names=()) -> list:
    """The usual param group without weight decay: ``[{"params": [...], "weight_decay": 0.0}]`` with every trainable
    parameter of ``module`` that has ``p.dim() <= 1`` (biases, normalisation weights) or whose name (as in
    ``module.named_parameters()``) is in ``names``.  Pass it, with any groups of your own, as ``BnetDDP(param_groups=...)``."""
    names = set(names)
    named = dict(module.named_parameters())
    unknown = names - set(named)
    if unknown:
        raise ValueError(f"no_weight_decay_groups: {sorted(unknown)} are not parameters of the module")
    return [{"params": [p for n, p in named.items() if p.requires_grad and (p.dim() <= 1 or n in names)], "weight_decay": 0.0}]


def _check_group_value(key: str, v) -> float:
    try:
        v = float(v)
    except (TypeError, ValueError):
        raise ValueError(f"param group {key!r} must be a number (got {v!r})") from None
    if not 0.0 <= v < math.inf:           # (False for NaN as well)
        raise ValueError(f"param group {key!r} must be finite and >= 0 (got {v})")
    return v


def _parse_param_groups(param_groups, params):
    """(group of every trainable parameter, lr_scale per group, weight_decay per group or None) from the user's list of
    dicts; the parameters no group lists form the default group, last.  Raises ValueError."""
    if isinstance(param_groups, dict) or not isinstance(param_groups, (list, tuple)):
        raise ValueError("param_groups must be a list of dicts, as torch.optim takes them")
    index = {id(p): i for i, p in enumerate(params)}
    group_of = [None] * len(params)
    scales, wds = [], []
    for k, g in enumerate(param_groups):
        if not isinstance(g, dict):
            raise ValueError(f"param group {k} is not a dict")
        extra = set(g) - {"params", "lr_scale", "weight_decay"}
        if "lr" in extra:
            raise ValueError(f"param group {k} sets 'lr': give a multiplier of the engine's lr as 'lr_scale' instead, so "
                             "that set_lr and a schedule move every group")
        if extra:
            raise ValueError(f"param group {k} has unknown keys {sorted(extra)}: a group takes 'params', 'lr_scale' and "
                             "'weight_decay' (the other hyper-parameters are the engine's)")
        if "params" not in g:
            raise ValueError(f"param group {k} has no 'params'")
        ps = g["params"]
        ps = [ps] if isinstance(ps, torch.Tensor) else list(ps)
        if not ps:
            raise ValueError(f"param group {k} has no parameters")
        for p in ps:
            i = index.get(id(p))
            if i is None or params[i] is not p:
                raise ValueError(f"param group {k} lists a tensor that is not a trainable parameter of the module")
            if group_of[i] is not None:
                raise ValueError(f"a parameter is in param groups {group_of[i]} and {k}")
            group_of[i] = k
        scales.append(_check_group_value("lr_scale", g.get("lr_scale", 1.0)))
        wds.append(_check_group_value("weight_decay", g["weight_decay"]) if "weight_decay" in g else None)
    if any(g is None for g in group_of):
        group_of = [len(scales) if g is None else g for g in group_of]
        scales.append(1.0)
        wds.append(None)
    if len(scales) > GROUPS_MAX:
        raise ValueError(f"{len(scales)} param groups (the default group included): the kernels take at most {GROUPS_MAX}")
    return group_of, scales, wds


def _torch_optimizer_kind(groups) -> str:
    """"adamw" or "sgd" for the param groups of a torch.optim.AdamW / SGD state_dict(); ValueError for anything else."""
    g = groups[0] if groups else {}
    if "betas" in g and "amsgrad" in g and g.get("decoupled_weight_decay", True):
        return "adamw"
    if "momentum" in g and "dampening" in g and "nesterov" in g:
        return "sgd"
    raise ValueError(f"not a torch.optim.SGD or AdamW state (param group keys {sorted(g)}); the engine fuses SGD, AdamW "
                     "and LARS")


def _check_max_norm(v) -> float:
    v = float(v)
    if not v > 0.0:                       # (False for NaN as well)
        raise ValueError(f"max_grad_norm must be > 0 or inf (got {v}); only the L2 norm is offered")
    return v


def _check_ema_decay(v) -> float:
    try:
        v = float(v)
    except (TypeError, ValueError):
        raise ValueError(f"ema_decay must be a number in [0, 1] (got {v!r})") from None
    if not 0.0 <= v <= 1.0:               # (False for NaN as well)
        raise ValueError(f"ema_decay must be in [0, 1] (got {v})")
    return v


class _Bucket:
    __slots__ = ("params", "start", "numel", "ready", "grad", "param", "state", "scratch", "partial", "launched", "ema",
                 "gsegs")

    def __init__(self):
        self.params = []
        self.start = 0
        self.numel = 0
        self.ready = 0
        self.scratch = None          # staged step: this rank's fp32 shard of the rank-summed (accumulated) gradient
        self.partial = None          # staged step: the bucket's row of per-CTA sums of squares
        self.launched = False        # staged step: stage 1 ran for this bucket in the current step (the scratch holds data)
        self.ema = None              # EMA of the master shard (fp32, same layout), kept apart from the optimizer's state
        self.gsegs = None            # parameter groups: the validated group segment table of this rank's shard

    @property
    def master(self) -> torch.Tensor:
        return self.state[0]


class BnetDDP(torch.nn.Module):
    """Wraps ``module``; owns the optimizer, fused into the collective: ``optimizer="sgd"`` (SGD with momentum and L2
    weight decay), ``"adamw"`` (``torch.optim.AdamW`` with ``betas``, ``eps`` and decoupled ``weight_decay``;
    AMSGrad and ``maximize`` are not offered) or ``"lars"``.

    ``"lars"``: layer-wise adaptive rate scaling, as NVIDIA Apex's ``LARC(clip=False)`` around ``torch.optim.SGD``
    (``momentum``, no dampening or Nesterov).  Every parameter tensor ``p`` with ``p.dim() > 1`` takes the trust ratio
    ``t = trust_coefficient * |p| / (|g| + weight_decay * |p| + eps)`` of its whole-tensor norms (``t = 1`` and no weight
    decay when either norm is 0, as in Apex) and steps with ``buf = momentum * buf + t * (g + weight_decay * p)``; biases and normalisation weights
    (``p.dim() <= 1``) take ``g`` alone, as in MLPerf's ResNet-50.  ``g`` is the mean gradient (clipped first when
    ``max_grad_norm`` is set).  The step is always staged; ``last_trust_ratios`` gives every tensor's ``t``.

    bucket_mb sizes buckets for launch latency and overlap (NVSwitch: no per-link bound).

    max_grad_norm: clip the mean gradient by its global L2 norm before the update, as
    ``torch.nn.utils.clip_grad_norm_(params, max_grad_norm)`` does (``inf`` computes the norm and never clips).  The step
    then runs in three stages: per bucket from the gradient hook, reduce into an fp32 scratch and sum squares; once per
    step, the norm and the coefficient; per bucket, the update from the scratch.  ``None`` keeps the one-kernel step.

    accumulation_steps: gradient accumulation over k micro-batches per optimizer step.  ``train_step`` splits its batch
    along dim 0 into k equal micro-batches, runs k forward/backward passes and one update, and returns the mean of the k
    losses.  Every micro-batch's gradients are reduced over the ranks while its backward runs and summed in this rank's
    fp32 scratch shard; the update (and clipping) runs once, on the k-th ``finish_step``, with the gradient scaled by
    1/(world * k): the gradient of the mean loss over the global batch.  In a loop of your own, call
    ``loss.backward(); engine.finish_step()`` once per micro-batch with the UNSCALED micro-batch loss (the mean over the
    micro-batch) -- do not divide it by k, the engine does that.  ``micro_step`` tells where in the step you are.
    BatchNorm statistics are per micro-batch, as with accumulation in torch.  ``1`` keeps the single-batch step.

    ema_decay: keep an exponential moving average of the fp32 master weights, as
    ``torch.optim.swa_utils.AveragedModel(module, multi_avg_fn=get_ema_multi_avg_fn(ema_decay), use_buffers=False)``
    with ``update_parameters`` called after every ``ema_every``-th optimizer step (steps counted from 1): the first
    update copies the masters, later ones take ``torch.lerp(ema, master, 1 - ema_decay)``.  Each rank keeps the EMA of
    its own master shards, and the update runs on the device behind the step's last update, so a captured CUDA graph
    decides on its own which steps update.  Buffers (BatchNorm statistics) are not averaged.  Evaluate or save the
    averaged model inside ``with engine.ema_parameters():``; ``set_ema_decay`` and ``reset_ema`` change it between steps.
    ``None`` keeps no EMA.

    param_groups: per-group learning rate and weight decay for ``"sgd"`` and ``"adamw"``, as torch.optim's param groups:
    a list of dicts with ``"params"`` (trainable parameters of ``module``), optionally ``"lr_scale"`` (>= 0, default 1:
    the group's lr is ``lr * lr_scale``) and ``"weight_decay"`` (>= 0, fixed for the group; without it the group follows
    the engine's ``weight_decay``).  Parameters no group lists form a default group, last.  At most 64 groups, the default
    one included.  ``no_weight_decay_groups(module)`` gives the usual group of biases and normalisation weights without
    decay.  Groups change neither the buckets nor the state layout; ``set_lr`` moves every group's lr through its scale
    and ``set_param_group`` changes one group, both without re-capturing a CUDA graph.  ``None`` keeps one lr and one
    weight decay for every parameter.
    """

    def __init__(self, module: torch.nn.Module, lr: float = 0.01, momentum: float | None = None, weight_decay: float = 0.0,
                 bucket_mb: float = 64.0, comm: SymmComm | None = None, extra_heap_bytes: int = 64 << 20,
                 nblocks: int = 0, group=None, optimizer: str = "sgd", betas: tuple[float, float] = (0.9, 0.999),
                 eps: float = 1e-8, amsgrad: bool = False, maximize: bool = False, max_grad_norm: float | None = None,
                 accumulation_steps: int = 1, trust_coefficient: float = 0.001, ema_decay: float | None = None,
                 ema_every: int = 1, param_groups: list | None = None):
        super().__init__()
        if ema_decay is not None:
            ema_decay = _check_ema_decay(ema_decay)
        if isinstance(ema_every, bool) or not isinstance(ema_every, int) or not 1 <= ema_every <= 1 << 24:
            # (the device block counts in floats, exact up to 2^24)
            raise ValueError(f"ema_every must be an int in [1, 2^24] (got {ema_every!r})")
        if isinstance(accumulation_steps, bool) or not isinstance(accumulation_steps, int) or accumulation_steps < 1:
            raise ValueError(f"accumulation_steps must be an int >= 1 (got {accumulation_steps!r})")
        if max_grad_norm is not None:
            max_grad_norm = _check_max_norm(max_grad_norm)
        if optimizer not in ("sgd", "adamw", "lars"):
            raise ValueError(f"unknown optimizer {optimizer!r}: BnetDDP fuses 'sgd', 'adamw' or 'lars'")
        if amsgrad or maximize:
            raise ValueError("the fused optimizers offer neither amsgrad nor maximize")
        if optimizer == "lars":
            trust_coefficient, eps = float(trust_coefficient), float(eps)
            if not trust_coefficient > 0.0 or not eps >= 0.0:
                raise ValueError(f"LARS needs trust_coefficient > 0 and eps >= 0 (got {trust_coefficient}, {eps})")
            self.trust_coefficient, self.eps = trust_coefficient, eps
        if optimizer == "adamw":
            if momentum is not None:
                raise ValueError("AdamW has no momentum argument; use betas")
            betas = (float(betas[0]), float(betas[1]))
            if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0) or not eps >= 0.0:
                raise ValueError(f"AdamW needs 0 <= beta < 1 and eps >= 0 (got betas={betas}, eps={eps})")
            self.betas, self.eps = betas, float(eps)
        elif momentum is None:
            momentum = 0.9
        self.optimizer = optimizer
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
        self._groups = None
        if param_groups is not None:
            if optimizer == "lars":
                raise ValueError("param_groups are offered for 'sgd' and 'adamw'; LARS excludes p.dim() <= 1 tensors itself")
            self._group_of, self._group_scale, self._group_wd = _parse_param_groups(param_groups, params)
        self._params = params
        self.dtype = dtype
        es = params[0].element_size()
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        plan, total = plan_buckets([p.numel() for p in params], es, world, bucket_mb)
        self._plan = plan                # (the full optimizer state dict maps shards to parameters through it)
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
        self.accumulation_steps = accumulation_steps
        self._micro = 0
        # the mean gradient over the global batch: world ranks times k micro-batches (for k = 1 exactly 1/world, as before)
        self._grad_scale = 1.0 / (comm.world * accumulation_steps)
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
        # fp32 master weights + optimizer state (momentum, or AdamW's two moments) for this rank's shard of every bucket
        for b in self.buckets:
            b.grad = self.flat_grad[b.start:b.start + b.numel]
            b.param = self.flat_param[b.start:b.start + b.numel]
            shard = b.numel // comm.world
            master = b.param[comm.rank * shard:(comm.rank + 1) * shard].float().contiguous()
            if ema_decay is not None and dtype == torch.float32:
                master = master.clone()   # (else a view of the parameters, which ema_parameters() overwrites)
            b.state = (master,) + tuple(torch.zeros_like(master) for _ in _STATE_NAMES[optimizer][1:])
        # AdamW and LARS always read their hyper-parameters (and AdamW its step count) from device memory
        # (csrc/cuda/optim_body.cuh); SGD passes them as launch arguments until the first set_lr
        self._hp = None
        if optimizer == "adamw":
            self._hp = torch.tensor(self._adamw_hp(0), dtype=torch.float32, device=dev)
        elif optimizer == "lars":
            self._hp = torch.tensor(self._lars_hp(), dtype=torch.float32, device=dev)
        # the staged step (gradient clipping, gradient accumulation, or both): per bucket an fp32 scratch shard and a row
        # of per-CTA partial sums of squares.  Clipping adds one exchange area in the heap (same offset on every rank) and
        # the device block {max_norm, total_norm, clip_coef, reserved}; accumulation without clipping updates through the
        # constant block {inf, 0, 1, 0} instead (clip_coef exactly 1).
        self._clip = None
        # (LARS needs every tensor's whole norm before any of it is updated: always staged)
        self._staged = max_grad_norm is not None or accumulation_steps > 1 or optimizer == "lars"
        if self._staged:
            from .comm import CLIP_ROW

            self._partials = torch.zeros(len(self.buckets), CLIP_ROW, dtype=torch.float64, device=dev)
            for b, row in zip(self.buckets, self._partials):
                b.scratch, b.partial = torch.zeros_like(b.master), row
        if max_grad_norm is not None:
            self._xchg = comm.alloc(comm.world, torch.float64)
            self._clip = torch.tensor([max_grad_norm, 0.0, 0.0, 0.0], dtype=torch.float32, device=dev)
        elif self._staged:
            self._coef_one = torch.tensor([float("inf"), 0.0, 1.0, 0.0], dtype=torch.float32, device=dev)
        self.max_grad_norm = max_grad_norm
        if optimizer == "lars":
            self._lars_setup(params, plan, es, dev)
        if param_groups is not None:
            self._groups_setup(params, plan, es, dev)
        # the EMA of the master shards, starting as their copy (AveragedModel deep-copies the model), and its device block
        self.ema_decay, self.ema_every, self._ema, self._in_ema = ema_decay, ema_every, None, False
        if ema_decay is not None:
            for b in self.buckets:
                b.ema = b.master.clone()
            self._ema = torch.tensor(self._ema_block(0, 0), dtype=torch.float32, device=dev)
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
        if self._staged:                         # staged step, stage 1: reduce into the scratch, sum of squares
            # the bucket's first contribution in this step stores, every later micro-batch's adds to it
            stage1 = self.comm.fused_accum_reduce_norm if b.launched else self.comm.fused_clip_reduce_norm
            stage1(b.grad, b.scratch, b.partial, channel=0, nblocks=self.nblocks, stream=self.comm_stream)
            b.launched = True
        elif self._groups is not None:
            step = self.comm.fused_allreduce_adamw_groups if self.optimizer == "adamw" else self.comm.fused_allreduce_sgd_groups
            step(b.grad, b.param, *b.state, self._hp, self._groups, b.gsegs, zero_grads=True, channel=0, nblocks=self.nblocks,
                 stream=self.comm_stream)
        elif self.optimizer == "adamw":
            self.comm.fused_allreduce_adamw(b.grad, b.param, *b.state, self._hp, zero_grads=True, channel=0,
                                            nblocks=self.nblocks, stream=self.comm_stream)
        else:
            self.comm.fused_allreduce_sgd(b.grad, b.param, *b.state, self.lr, self.momentum, self.weight_decay,
                                          zero_grads=True, channel=0, nblocks=self.nblocks, stream=self.comm_stream,
                                          hp=self._hp)
        b.ready = 0
        self._inflight = True

    def finish_step(self):
        """Make the updated parameters visible to the compute stream (call after backward).  With
        ``accumulation_steps=k``, call it after every micro-batch's backward: the first k-1 calls only reduce that
        micro-batch's gradients into the scratch, the k-th also updates."""
        self._check_not_in_ema("finish_step")
        for b in self.buckets:
            if b.ready:                           # parameters that got no gradient this step
                self._launch(b)
        if self.accumulation_steps > 1:
            self._micro += 1
            if self._micro < self.accumulation_steps:
                # the next backward writes into gradient slices that this micro-batch's stage 1 zeroes
                if self._inflight:
                    torch.cuda.current_stream().wait_stream(self.comm_stream)
                return
            self._micro = 0
        if self._inflight:
            if self._staged:
                self._staged_update()
            if self._ema is not None:
                # behind the step's last update, on the comm stream: every bucket's EMA shard (the kernels skip the
                # steps that are not EMA steps on the device), then the step count
                for b in self.buckets:
                    self.comm.ema_update(b.master, b.ema, self._ema, nblocks=self.nblocks, stream=self.comm_stream)
                self.comm.ema_advance(self._ema, stream=self.comm_stream)
            if self.optimizer == "adamw":
                # one optimizer step taken: advance the step count the kernels read, behind this step's last bucket
                # (on the comm stream, so a captured step replays it)
                with torch.cuda.stream(self.comm_stream):
                    self._hp[self._HP_STEP:self._HP_STEP + 1].add_(1.0)
            torch.cuda.current_stream().wait_stream(self.comm_stream)
            self._inflight = False

    def _staged_update(self):
        """Stages 2 and 3 of the staged step (clipping and/or accumulation), on the comm stream behind every bucket's
        stage 1, once per optimizer step."""
        # Behind the whole backward: stage 2's rank barrier then also means that every rank's backward is done, which
        # is what lets stage 3 write new parameters into the peers without an opening barrier of its own.
        self.comm_stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.comm_stream):
            for b in self.buckets:
                if not b.launched:                # no gradient at all this step: no update, and nothing in the norm
                    b.partial.zero_()
        if self._clip is not None:
            self.comm.fused_clip_coef(self._partials, self._xchg, self._clip, grad_scale=self._grad_scale, channel=0,
                                      stream=self.comm_stream)
            coef = self._clip
        else:
            coef = self._coef_one
        if self.optimizer == "lars":
            self._lars_update(coef)
            return
        if self._clip is None:
            # accumulation without clipping: only the barrier, and a coefficient of exactly 1.  (Not the coefficient
            # kernel at max_norm = inf: that turns a NaN norm into a NaN coefficient for every element, where an
            # unclipped torch step poisons only the NaN elements.)
            self.comm.barrier(channel=0, stream=self.comm_stream)
        for b in self.buckets:
            if not b.launched:
                continue
            if self._groups is not None:
                apply = self.comm.fused_clip_apply_adamw_groups if self.optimizer == "adamw" else self.comm.fused_clip_apply_sgd_groups
                apply(b.param, b.scratch, coef, *b.state, self._hp, self._groups, b.gsegs, channel=0, nblocks=self.nblocks,
                      stream=self.comm_stream)
            elif self.optimizer == "adamw":
                self.comm.fused_clip_apply_adamw(b.param, b.scratch, coef, *b.state, self._hp, channel=0,
                                                 nblocks=self.nblocks, stream=self.comm_stream)
            else:
                self.comm.fused_clip_apply_sgd(b.param, b.scratch, coef, *b.state, self.lr, self.momentum,
                                               self.weight_decay, self._grad_scale, channel=0, nblocks=self.nblocks,
                                               stream=self.comm_stream, hp=self._hp)
            b.launched = False

    # ------------------------------------------------------------------ parameter groups
    def _groups_setup(self, params, plan, es, dev):
        """Per bucket the validated group segment table of this rank's shard; the device group table; for SGD the
        4-float block the grouped kernels read momentum and gradient scale from (their lr and weight decay are unused)."""
        numels = [p.numel() for p in params]
        G = len(self._group_scale)
        for b, (start, numel, members) in zip(self.buckets, plan):
            table = group_segments(members, numels, self._group_of, start, numel, es, self.comm.world, self.comm.rank)
            b.gsegs = self.comm.group_segments(table, numel // self.comm.world * es // 16, G)
        self._groups = torch.zeros(G, 4, dtype=torch.float32, device=dev)
        if self.optimizer == "sgd":
            self._hp = torch.tensor([self.lr, self.momentum, self.weight_decay, self._grad_scale], dtype=torch.float32,
                                    device=dev)
        self._write_groups()

    def _write_groups(self) -> None:
        """The device group table {lr, weight_decay, 0, 0} per group from the host values: lr = engine lr * lr_scale in
        double, rounded once to fp32 (as torch rounds a Python-float group lr)."""
        if self._groups is None:
            return
        rows = [[self.lr * s, self.weight_decay if wd is None else wd, 0.0, 0.0] for s, wd in zip(self._group_scale, self._group_wd)]
        self._groups.copy_(torch.tensor(rows, dtype=torch.float64).to(torch.float32))

    def _require_groups(self, what: str) -> None:
        if self._groups is None:
            raise ValueError(f"cannot {what}: the engine has no param groups (build it with param_groups=...)")

    @property
    def param_groups(self) -> list | None:
        """Copies of the parameter groups, default group last: ``{"params", "lr_scale", "weight_decay", "lr"}`` with the
        effective values (a group that follows the engine shows the engine's weight decay).  Changing them changes
        nothing; use ``set_lr`` and ``set_param_group``.  ``None`` without groups."""
        if self._groups is None:
            return None
        return [{"params": [p for p, g in zip(self._params, self._group_of) if g == k], "lr_scale": s,
                 "weight_decay": self.weight_decay if wd is None else wd, "lr": self.lr * s}
                for k, (s, wd) in enumerate(zip(self._group_scale, self._group_wd))]

    def set_param_group(self, i: int, lr_scale: float | None = None, weight_decay: float | None = None) -> None:
        """Change group ``i``'s lr_scale and/or weight decay (a fixed weight decay from then on) between steps.  Only the
        device group table is rewritten, so a captured CUDA graph follows without being re-captured."""
        self._require_groups("set a param group")
        if isinstance(i, bool) or not isinstance(i, int) or not 0 <= i < len(self._group_scale):
            raise ValueError(f"param group {i!r} does not exist (the engine has {len(self._group_scale)})")
        s = self._group_scale[i] if lr_scale is None else _check_group_value("lr_scale", lr_scale)
        wd = self._group_wd[i] if weight_decay is None else _check_group_value("weight_decay", weight_decay)
        self._group_scale[i], self._group_wd[i] = s, wd
        self._write_groups()

    def _groups_state(self) -> list:
        return [{"params": [j for j, g in enumerate(self._group_of) if g == k], "lr_scale": s, "weight_decay": wd}
                for k, (s, wd) in enumerate(zip(self._group_scale, self._group_wd))]

    # ------------------------------------------------------------------ LARS
    def _lars_setup(self, params, plan, es, dev):
        """Per bucket the validated segment table of this rank's shard and its norm slots; per tensor its slot range and
        whether it is excluded; the exchange area in the heap, the update scalars and the trust ratios."""
        comm, T = self.comm, len(params)
        numels = [p.numel() for p in params]
        tensors = [[0, 0, int(p.dim() <= 1), 0] for p in params]
        self._lars_segs, self._lars_base, base = [], [], 0
        for b, (start, numel, members) in zip(self.buckets, plan):
            table = lars_segments(members, numels, start, numel, es, comm.world, comm.rank)
            segs = comm.lars_segments(table, numel // comm.world * es // 16, T)
            for vec0, nvec, pi, slot0 in table:
                if tensors[pi][1]:
                    raise AssertionError(f"tensor {pi} has two segments on one rank")
                tensors[pi][:2] = [base + slot0, (nvec + LARS_CHUNK - 1) // LARS_CHUNK]
            self._lars_segs.append(segs)
            self._lars_base.append(base)
            base += sum((nvec + LARS_CHUNK - 1) // LARS_CHUNK for _, nvec, _, _ in table)
        self._lars_base.append(base)
        self._lars_slots = torch.zeros(base, 2, dtype=torch.float64, device=dev)
        self._lars_tensors = comm.lars_tensors(tensors, base)
        self._lars_xchg = comm.alloc(2 * comm.world * T, torch.float64)
        self._lars_scal = torch.zeros(T, 2, dtype=torch.float32, device=dev)
        self._lars_trust = torch.ones(T, dtype=torch.float32, device=dev)

    def _lars_update(self, coef):
        """The LARS stages after the clipping coefficient: norms per launched bucket, the trust kernel (whose barrier is
        the step's when there is no coefficient kernel), the update per launched bucket."""
        st = self.comm_stream
        for k, b in enumerate(self.buckets):
            slots = self._lars_slots[self._lars_base[k]:self._lars_base[k + 1]]
            if b.launched:
                self.comm.fused_lars_norm(b.master, b.scratch, self._lars_segs[k], slots, self.dtype, nblocks=self.nblocks,
                                          stream=st)
            else:
                with torch.cuda.stream(st):
                    slots.zero_()                 # no gradient this step: its tensors' ratios read 1, and no update
        self.comm.fused_lars_trust(self._lars_slots, self._lars_tensors, self._lars_xchg, coef, self._hp, self._lars_scal,
                                   self._lars_trust, channel=0, stream=st)
        for k, b in enumerate(self.buckets):
            if not b.launched:
                continue
            self.comm.fused_lars_apply(b.param, b.scratch, self._lars_segs[k], self._lars_scal, self._hp, *b.state, channel=0,
                                       nblocks=self.nblocks, stream=st)
            b.launched = False

    def _lars_hp(self) -> list:
        return [self.lr, self.momentum, self.weight_decay, self._grad_scale, self.trust_coefficient, self.eps, 0.0, 0.0]

    @property
    def last_trust_ratios(self) -> torch.Tensor | None:
        """LARS: the trust ratio of every trainable parameter of the most recent step, in ``module.parameters()`` order
        (1 for the excluded ``p.dim() <= 1`` tensors and for tensors without a gradient in the step), as a new fp32
        tensor on the device.  ``None`` for the other optimizers."""
        return None if self.optimizer != "lars" else self._lars_trust.clone()

    # ------------------------------------------------------------------ user API
    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def _eager_step(self, inputs, targets, loss_fn):
        k = self.accumulation_steps
        if k == 1:
            out = self.module(inputs)
            loss = loss_fn(out.float(), targets)
            loss.backward()
            self.finish_step()
            return loss.detach()
        # k micro-batches: equal views along dim 0 (the slices of a channels_last batch are channels_last)
        losses = []
        for x, y in zip(inputs.split(inputs.shape[0] // k), targets.split(targets.shape[0] // k)):
            loss = loss_fn(self.module(x).float(), y)
            loss.backward()
            self.finish_step()
            losses.append(loss.detach())
        return torch.stack(losses).mean()

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
            # optimizer state, the hyper-parameter block (AdamW's step count), the EMA shards and block, module buffers
            # (BatchNorm running statistics).  A (re)capture therefore leaves the training trajectory exactly where
            # eager mode would have it; checkpoint/resume stays step-exact.
            live = [self.flat_param] + [t for b in self.buckets for t in b.state]
            live += [b.ema for b in self.buckets if b.ema is not None]
            live += [t for t in self.module.buffers() if t.is_cuda and t.numel()]
            live += [t for t in (self._hp, self._clip, self._ema) if t is not None]
            saved = [t.clone() for t in live]
            for _ in range(2):
                self._eager_step(self._gx, self._gy, loss_fn)
            self._micro = 0                         # (two whole steps: back at the first micro-batch already)
            torch.cuda.current_stream().synchronize()
            if self.comm.world > 1:
                dist.barrier()                      # nobody restores while a peer's kernel still writes parameters
            for t, s in zip(live, saved):
                t.copy_(s)
            del live, saved
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
        """forward + backward + fused all-reduce/optimizer.  Returns the (device) loss tensor.  With
        ``accumulation_steps=k``: k micro-batches of ``inputs.shape[0] // k`` samples and one update; the loss returned
        is the mean of the k micro-batch losses."""
        k = self.accumulation_steps
        self._check_not_in_ema("train_step")
        if self._micro:
            raise ValueError(f"train_step called in the middle of an accumulation step (micro_step={self._micro}): "
                             "finish that step with backward + finish_step first")
        if k > 1 and (inputs.shape[0] % k or targets.shape[0] != inputs.shape[0]):
            raise ValueError(f"a batch of {inputs.shape[0]} inputs / {targets.shape[0]} targets does not split into "
                             f"accumulation_steps={k} equal micro-batches")
        loss_fn = loss_fn or torch.nn.functional.cross_entropy
        if not getattr(self, "_use_graph", False):
            return self._eager_step(inputs, targets, loss_fn)
        from ..ops import fused_nn

        # with the hyper-parameters in device memory (after the first set_lr) the captured step does not depend on them
        hpkey = "device" if self._hp is not None else (self.lr, self.momentum, self.weight_decay)
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
    # weights and momentum (SGD) or exp_avg / exp_avg_sq (AdamW, which also saves its step count) of every bucket.
    def _check_step_boundary(self, what: str) -> None:
        if self._micro:
            raise ValueError(f"cannot {what} in the middle of an accumulation step (micro_step={self._micro}): the "
                             "scratch holds a partial gradient sum that is not saved")

    def optimizer_state_dict(self) -> dict:
        self._check_step_boundary("save the optimizer state")
        if self.optimizer == "adamw":
            head = {"optimizer": "adamw", "lr": self.lr, "betas": self.betas, "eps": self.eps,
                    "weight_decay": self.weight_decay, "step": int(self._hp[self._HP_STEP].item())}
        elif self.optimizer == "lars":
            head = {"optimizer": "lars", "lr": self.lr, "momentum": self.momentum, "weight_decay": self.weight_decay,
                    "trust_coefficient": self.trust_coefficient, "eps": self.eps}
        else:
            head = {"lr": self.lr, "momentum": self.momentum, "weight_decay": self.weight_decay}
        if self._groups is not None:
            head["param_groups"] = self._groups_state()
        names = _STATE_NAMES[self.optimizer]
        buckets = [{k: t.detach().cpu() for k, t in zip(names, b.state)} for b in self.buckets]
        if self._ema is not None:
            step, n_averaged = (int(v) for v in self._ema[self._EMA_STEP:].tolist())
            head.update(ema_decay=self.ema_decay, ema_every=self.ema_every, ema_step=step, ema_n_averaged=n_averaged)
            for d, b in zip(buckets, self.buckets):
                d["ema"] = b.ema.detach().cpu()
        return {**head, "world": self.comm.world, "rank": self.comm.rank, "buckets": buckets}

    def load_optimizer_state_dict(self, state: dict) -> None:
        self._check_step_boundary("load an optimizer state")
        kind = state.get("optimizer", "sgd")
        if kind != self.optimizer:
            raise ValueError(f"optimizer state of {kind!r} cannot be loaded into a {self.optimizer!r} engine")
        if state["world"] != self.comm.world or state["rank"] != self.comm.rank or len(state["buckets"]) != len(self.buckets):
            raise ValueError("optimizer state was saved for a different world size / rank / bucket layout")
        has_ema = "ema_decay" in state
        if has_ema and self._ema is None:
            raise ValueError("the optimizer state holds an EMA of the weights, which this engine would drop: build it with "
                             "ema_decay=... to load it")
        for b, s in zip(self.buckets, state["buckets"]):
            if s["master"].shape != b.master.shape or (has_ema and s["ema"].shape != b.master.shape):
                raise ValueError("optimizer state shard does not match this bucket")
        groups = state.get("param_groups")
        if (groups is None) != (self._groups is None):
            raise ValueError("the optimizer state and this engine disagree on param groups: one has them, the other not")
        if groups is not None:
            if [list(g["params"]) for g in groups] != [g["params"] for g in self._groups_state()]:
                raise ValueError("the optimizer state's param groups hold other parameters than this engine's")
            scales = [_check_group_value("lr_scale", g["lr_scale"]) for g in groups]
            wds = [None if g["weight_decay"] is None else _check_group_value("weight_decay", g["weight_decay"]) for g in groups]
        else:
            scales = wds = None
        for b, s in zip(self.buckets, state["buckets"]):
            for k, t in zip(_STATE_NAMES[self.optimizer], b.state):
                t.copy_(s[k])
        if self._ema is not None:
            # a state without an EMA (fine-tuning from a plain checkpoint): the EMA restarts from the loaded masters
            if has_ema:
                self.ema_decay, self.ema_every = _check_ema_decay(state["ema_decay"]), int(state["ema_every"])
            for b, s in zip(self.buckets, state["buckets"]):
                b.ema.copy_(s["ema"] if has_ema else b.master)
            counts = (state["ema_step"], state["ema_n_averaged"]) if has_ema else (0, 0)
            self._ema.copy_(torch.tensor(self._ema_block(*counts), dtype=torch.float32))
        self._restore_hyper(state["lr"], state["weight_decay"], state, scales, wds, state.get("step", 0))

    # The layout-free format: torch.optim.Optimizer.state_dict()'s layout, with no trace of the world size, the rank or the
    # buckets, plus a "bnet" entry for what torch has no slot for.  Index i numbers the trainable parameters group by
    # group in the order of `param_groups` (default group last), module order within a group: the numbering torch.optim
    # gives when it is built from those groups.
    _FULL_VERSION = 1
    _TORCH_STATE = {"sgd": ("momentum_buffer",), "lars": ("momentum_buffer",), "adamw": ("exp_avg", "exp_avg_sq")}

    def _check_checkpoint_call(self, what: str) -> None:
        self._check_step_boundary(what)
        if self._in_ema:
            raise ValueError(f"cannot {what} inside ema_parameters(): the parameters hold the EMA weights")
        if self.flat_param.is_cuda and torch.cuda.is_current_stream_capturing():
            raise ValueError(f"cannot {what} inside a CUDA graph capture")

    def _torch_order(self) -> list:
        """The engine's parameter index (module order) of every torch.optim index."""
        if self._groups is None:
            return list(range(len(self._params)))
        return [j for k in range(len(self._group_scale)) for j, g in enumerate(self._group_of) if g == k]

    def _torch_groups(self) -> list:
        """torch.optim's param groups with the effective values, each with its ``lr_scale``, ``params`` as torch indices."""
        if self.optimizer == "adamw":
            hyper = {"betas": tuple(self.betas), "eps": self.eps, "amsgrad": False, "maximize": False,
                     "decoupled_weight_decay": True}     # (without it torch.optim.AdamW.load_state_dict turns into Adam)
        else:
            hyper = {"momentum": self.momentum, "dampening": 0, "nesterov": False, "maximize": False}
            if self.optimizer == "lars":
                hyper.update(trust_coefficient=self.trust_coefficient, eps=self.eps)
        if self._groups is None:
            groups = [(len(self._params), 1.0, self.weight_decay)]
        else:
            groups = [(self._group_of.count(k), s, self.weight_decay if wd is None else wd)
                      for k, (s, wd) in enumerate(zip(self._group_scale, self._group_wd))]
        out, i = [], 0
        for n, s, wd in groups:
            out.append({"lr": self.lr * s, **hyper, "weight_decay": wd, "lr_scale": s, "params": list(range(i, i + n))})
            i += n
        return out

    def full_optimizer_state_dict(self) -> dict | None:
        """The whole optimizer state, independent of the world size and the bucket layout, in the layout of
        ``torch.optim.Optimizer.state_dict()`` (see docs/API.md).  Collective: every rank calls it; rank 0 gets the dict
        (tensors in host memory), the other ranks ``None``.  The shards travel bucket by bucket, one source rank at a
        time, through the heap's broadcast, so no rank holds more than one shard of one bucket on the device."""
        self._check_checkpoint_call("save the optimizer state")
        world, rank = self.comm.world, self.comm.rank
        names = _STATE_NAMES[self.optimizer] + (("ema",) if self._ema is not None else ())
        step = int(self._hp[self._HP_STEP].item()) if self.optimizer == "adamw" else None
        counts = [int(v) for v in self._ema[self._EMA_STEP:].tolist()] if self._ema is not None else None
        fulls = flats = pieces = None
        if rank == 0:
            fulls = {n: [torch.empty_like(p, dtype=torch.float32, device="cpu") for p in self._params] for n in names}
            flats = {n: [memory_flat(t) for t in ts] for n, ts in fulls.items()}
            numels = [p.numel() for p in self._params]
            pieces = [shard_pieces(self._plan, numels, world, r) for r in range(world)]
        for k, b in enumerate(self.buckets):
            for n, t in zip(names, b.state + ((b.ema,) if b.ema is not None else ())):
                for src in range(world):
                    shard = t.detach()
                    if src != 0:                  # (collective: every rank takes part in every source's broadcast)
                        shard = shard.clone() if rank == src else torch.empty_like(t)
                        self.comm.broadcast_tensor(shard, src=src)
                    if rank == 0:                 # (each piece straight from the device into its host tensor)
                        full_from_shard(flats[n], pieces[src][k], shard)
        if rank != 0:
            return None
        order = self._torch_order()
        if self.optimizer == "adamw":
            state = {i: {"step": torch.tensor(float(step), dtype=torch.float32), "exp_avg": fulls["exp_avg"][j],
                         "exp_avg_sq": fulls["exp_avg_sq"][j]} for i, j in enumerate(order)}
        else:
            state = {i: {"momentum_buffer": fulls["momentum"][j]} for i, j in enumerate(order)}
        bnet = {"version": self._FULL_VERSION, "optimizer": self.optimizer, "lr": self.lr, "weight_decay": self.weight_decay,
                "group_weight_decay": None if self._groups is None else list(self._group_wd),
                "master": {i: fulls["master"][j] for i, j in enumerate(order)}}
        if step is not None:
            bnet["step"] = step
        if self._ema is not None:
            bnet.update(ema={i: fulls["ema"][j] for i, j in enumerate(order)}, ema_decay=self.ema_decay,
                        ema_every=self.ema_every, ema_step=counts[0], ema_n_averaged=counts[1])
        return {"state": state, "param_groups": self._torch_groups(), "bnet": bnet}

    def load_full_optimizer_state_dict(self, state: dict) -> None:
        """Load a dict of ``full_optimizer_state_dict`` (saved at any world size and ``bucket_mb``), or a plain
        ``torch.optim.SGD`` / ``AdamW`` ``state_dict()``.  Every rank calls it with the same dict and copies out its own
        shards; no communication.  Raises ValueError for a state the engine cannot represent (see docs/API.md)."""
        self._check_checkpoint_call("load an optimizer state")
        groups = list(state["param_groups"])
        bnet = state.get("bnet")
        ours = self._torch_groups()
        if bnet is None:
            kind = _torch_optimizer_kind(groups)
            if kind != self.optimizer:
                raise ValueError(f"a torch.optim {kind} state cannot be loaded into a {self.optimizer!r} engine")
            if self._groups is None and len(groups) > 1:
                raise ValueError(f"the torch.optim state has {len(groups)} param groups and this engine none: build it "
                                 "with the same param_groups")
        else:
            if bnet.get("version") != self._FULL_VERSION:
                raise ValueError(f"unknown full optimizer state version {bnet.get('version')!r}")
            kind = bnet["optimizer"]
            if kind != self.optimizer:
                raise ValueError(f"optimizer state of {kind!r} cannot be loaded into a {self.optimizer!r} engine")
            if (bnet["group_weight_decay"] is None) != (self._groups is None):
                raise ValueError("the optimizer state and this engine disagree on param groups: one has them, the other not")
            if "ema" in bnet and self._ema is None:
                raise ValueError("the optimizer state holds an EMA of the weights, which this engine would drop: build it "
                                 "with ema_decay=... to load it")
        if [list(g["params"]) for g in groups] != [g["params"] for g in ours]:
            raise ValueError("the optimizer state's param groups hold other parameters than this engine's")
        order = self._torch_order()
        per_param = state.get("state", {})
        values = {n: [None] * len(order) for n in self._TORCH_STATE[self.optimizer]}
        steps = set()
        for i, j in enumerate(order):
            entry = per_param.get(i) or {}
            for n in values:
                v = entry.get(n)
                if v is not None:
                    values[n][j] = self._check_full_shape(v, j, n)
            if self.optimizer == "adamw" and entry.get("step") is not None:
                steps.add(float(entry["step"]))
        if bnet is None:
            lr, wd, step, scales, wds = self._torch_hyper(groups, steps)
            master = ema = None
        else:
            lr, wd, step = bnet["lr"], bnet["weight_decay"], bnet.get("step", 0)
            scales = [_check_group_value("lr_scale", g["lr_scale"]) for g in groups]
            wds = [None if v is None else _check_group_value("weight_decay", v) for v in bnet["group_weight_decay"] or ()]
            master, ema = [None] * len(order), [None] * len(order) if "ema" in bnet else None
            for i, j in enumerate(order):
                master[j] = self._check_full_shape(bnet["master"][i], j, "master")
                if ema is not None:
                    ema[j] = self._check_full_shape(bnet["ema"][i], j, "ema")
        # everything is checked: from here on nothing raises
        numels = [p.numel() for p in self._params]
        for b, pieces in zip(self.buckets, shard_pieces(self._plan, numels, self.comm.world, self.comm.rank)):
            srcs = [master] + [values[n] for n in self._TORCH_STATE[self.optimizer]]
            if self._ema is not None:
                srcs.append(ema)
            for t, src in zip(b.state + ((b.ema,) if b.ema is not None else ()), srcs):
                if src is None:
                    continue                      # (masters from the parameters, an EMA from the masters: below)
                shard_from_full({pi: self._layout_flat(src[pi], pi) for pi, _, _, _ in pieces}, pieces, t)
        if master is None:
            self.sync_master_from_params()
        if self._ema is not None:
            counts = (0, 0)
            if ema is not None:
                self.ema_decay, self.ema_every = _check_ema_decay(bnet["ema_decay"]), int(bnet["ema_every"])
                counts = (bnet["ema_step"], bnet["ema_n_averaged"])
            else:
                for b in self.buckets:
                    b.ema.copy_(b.master)
            self._ema.copy_(torch.tensor(self._ema_block(*counts), dtype=torch.float32))
        self._restore_hyper(lr, wd, groups[-1], scales, wds, step)

    def _check_full_shape(self, v, j: int, what: str) -> torch.Tensor:
        p = self._params[j]
        if not isinstance(v, torch.Tensor) or tuple(v.shape) != tuple(p.shape):
            raise ValueError(f"the optimizer state's {what} of parameter {j} has shape "
                             f"{tuple(v.shape) if isinstance(v, torch.Tensor) else type(v).__name__}, the parameter "
                             f"{tuple(p.shape)}")
        return v

    def _layout_flat(self, v, pi: int) -> torch.Tensor:
        """``v`` (parameter ``pi``'s shape, any layout and device; None: zeros) as fp32 in the parameter's memory order."""
        p = self._params[pi]
        if v is None:
            return torch.zeros(p.numel(), dtype=torch.float32)
        if v.dtype != torch.float32 or v.stride() != p.stride():
            v = torch.empty_like(p, dtype=torch.float32, device=v.device).copy_(v)
        return memory_flat(v)

    def _torch_hyper(self, groups, steps):
        """(lr, weight decay, AdamW step, lr_scales, weight decays) from a torch.optim state's param groups and the step
        counts of its parameters.  Raises ValueError for what the fused optimizers cannot represent."""
        for g in groups:
            for key in ("nesterov", "amsgrad", "maximize"):
                if g.get(key, False):
                    raise ValueError(f"the torch.optim state sets {key}, which the fused optimizers do not offer")
            if g.get("dampening", 0) != 0:
                raise ValueError(f"the torch.optim state has dampening={g['dampening']}; the fused SGD has none")
        keys = ("betas", "eps") if self.optimizer == "adamw" else ("momentum",)
        for key in keys:
            if any(tuple(g[key]) != tuple(groups[0][key]) if key == "betas" else g[key] != groups[0][key] for g in groups):
                raise ValueError(f"the torch.optim state's param groups differ in {key}; the engine has one for all groups")
        if len(steps) > 1:
            raise ValueError(f"the torch.optim state's parameters are at different AdamW steps {sorted(steps)}; the "
                             "engine keeps one step count")
        lrs = [_check_group_value("lr", g["lr"]) for g in groups]
        wds = [_check_group_value("weight_decay", g["weight_decay"]) for g in groups]
        lr = lrs[-1]
        if lr == 0 and any(v > 0 for v in lrs):
            raise ValueError("the torch.optim state's last param group has lr 0 and another one not: the engine's lr is "
                             "the last group's and every group's lr a multiple of it")
        scales = [v / lr if lr else 1.0 for v in lrs]
        return lr, wds[-1], int(steps.pop()) if steps else 0, scales, wds

    def _restore_hyper(self, lr, weight_decay, group: dict, scales, wds, step: int) -> None:
        """Set the hyper-parameters (momentum / betas, eps and LARS's trust coefficient from the param group `group`) and
        refresh the device blocks, so that a captured CUDA graph follows."""
        self.lr, self.weight_decay = lr, weight_decay
        if self._groups is not None:
            self._group_scale, self._group_wd = scales, wds
        if self.optimizer == "adamw":
            self.betas, self.eps = tuple(group["betas"]), group["eps"]
            self._hp.copy_(torch.tensor(self._adamw_hp(step), dtype=torch.float32))
            self._write_groups()
            return
        self.momentum = group["momentum"]
        if self.optimizer == "lars":
            self.trust_coefficient, self.eps = group["trust_coefficient"], group["eps"]
            self._hp.copy_(torch.tensor(self._lars_hp(), dtype=torch.float32))
        elif self._hp is not None:
            self.set_lr(self.lr)              # hyper-parameters live in device memory: refresh them (and the group table)
        else:
            self._graph = None                # hyper-parameters are baked into a captured step

    def sync_master_from_params(self) -> None:
        """After module.load_state_dict(): rebuild the fp32 master shards from the (just loaded) parameters.  The EMA
        of the weights is left as it is; call ``reset_ema()`` as well to restart it from the loaded weights."""
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
        graph is re-captured once (here) and then follows the schedule with one tiny host→device write per change.
        AdamW and LARS read theirs from device memory from the start (no re-capture at all); AdamW has no momentum, and
        LARS's block also holds its trust coefficient and eps, fixed at construction."""
        if self.optimizer == "adamw":
            if momentum is not None:
                raise ValueError("AdamW has no momentum; its betas are fixed at construction")
            self.lr = float(lr)
            if weight_decay is not None:
                self.weight_decay = float(weight_decay)
            # everything but the step count, which the captured steps advance on the device
            self._hp[:self._HP_STEP].copy_(torch.tensor(self._adamw_hp(0)[:self._HP_STEP], dtype=torch.float32))
            self._write_groups()
            return
        self.lr = float(lr)
        if momentum is not None:
            self.momentum = float(momentum)
        if weight_decay is not None:
            self.weight_decay = float(weight_decay)
        vals = [self.lr, self.momentum, self.weight_decay, self._grad_scale]
        if self.optimizer == "lars":           # (the block has been in device memory since construction)
            self._hp.copy_(torch.tensor(self._lars_hp(), dtype=torch.float32))
            return
        if self._hp is None:
            self._hp = torch.tensor(vals, dtype=torch.float32, device=self.flat_param.device)
            self._graph = None
        else:
            self._hp.copy_(torch.tensor(vals, dtype=torch.float32), non_blocking=False)
        self._write_groups()                   # (every group's lr follows through its scale)

    def set_max_grad_norm(self, max_norm: float) -> None:
        """Change the clipping threshold of an engine built with ``max_grad_norm``.  The norm kernel reads it from
        device memory, so a captured CUDA graph follows it without being re-captured."""
        if self._clip is None:
            raise ValueError("gradient clipping is off: build the engine with max_grad_norm=... to enable it")
        self.max_grad_norm = _check_max_norm(max_norm)
        self._clip[:1].copy_(torch.tensor([self.max_grad_norm], dtype=torch.float32))

    @property
    def last_grad_norm(self) -> torch.Tensor | None:
        """The global L2 norm of the mean gradient before clipping in the most recent step (what ``clip_grad_norm_``
        returns), as a new 0-dim fp32 tensor on the device: a copy taken on the current stream, so tensors kept from
        earlier steps keep their values and reading one is the only synchronisation.  ``None`` without clipping."""
        return None if self._clip is None else self._clip[1].clone()

    # AdamW's hyper-parameter block: {lr, beta1, beta2, eps, weight_decay, grad_scale, step, reserved}
    _HP_STEP = 6

    # ------------------------------------------------------------------ exponential moving average of the weights
    # The EMA block (csrc/cuda/optim_body.cuh): {1 - decay, every, step, n_averaged}
    _EMA_STEP = 2

    def _ema_block(self, step: int, n_averaged: int) -> list:
        # 1 - decay in double, rounded once to fp32: the weight torch._foreach_lerp_ gets from get_ema_multi_avg_fn
        return [1.0 - self.ema_decay, float(self.ema_every), float(step), float(n_averaged)]

    def _require_ema(self, what: str) -> None:
        if self._ema is None:
            raise ValueError(f"cannot {what}: the engine keeps no EMA of the weights (build it with ema_decay=...)")

    def _check_not_in_ema(self, what: str) -> None:
        if self._in_ema:
            raise ValueError(f"{what} inside ema_parameters(): the parameters hold the EMA weights, not the trained ones")

    def set_ema_decay(self, decay: float) -> None:
        """Change the EMA's decay (a warm-up schedule, say).  The update kernels read it from device memory, so a
        captured CUDA graph follows it without being re-captured."""
        self._require_ema("set the EMA decay")
        self.ema_decay = _check_ema_decay(decay)
        self._ema[:1].copy_(torch.tensor([1.0 - self.ema_decay], dtype=torch.float32))

    def reset_ema(self) -> None:
        """Set the EMA's update count to 0 on the device, so that its next update copies the master weights (what
        ``model_ema.n_averaged.fill_(0)`` does for an ``AveragedModel``).  The step count goes on."""
        self._require_ema("reset the EMA")
        self._ema[self._EMA_STEP + 1:].zero_()

    @contextlib.contextmanager
    def ema_parameters(self):
        """Inside the block the module's parameters are the EMA weights, rounded to the parameter dtype, on every rank:
        for evaluation, or for ``module.state_dict()`` of the averaged model.  On exit they are the trained parameters
        again, bitwise.  Collective: every rank enters and leaves together.  ``train_step`` and ``finish_step`` raise
        inside it.  Yields the module."""
        self._require_ema("swap in the EMA weights")
        self._check_step_boundary("swap in the EMA weights")
        if self._in_ema:
            raise ValueError("ema_parameters() is already active")
        if self.flat_param.is_cuda and torch.cuda.is_current_stream_capturing():
            raise ValueError("ema_parameters() cannot run inside a CUDA graph capture")
        self._publish(lambda b: b.ema)
        self._in_ema = True
        try:
            yield self.module
        finally:
            self._in_ema = False
            self._publish(lambda b: b.master)

    def _publish(self, shard_of) -> None:
        """Every rank writes ``shard_of(bucket)`` (an fp32 shard laid out as the master), rounded to the parameter dtype
        as the update kernels round, into its part of every rank's parameters, on the current stream.  The opening
        barrier means every rank is done with its step and with reading the parameters; the closing one, that every
        rank's parameters are complete."""
        cur = torch.cuda.current_stream()
        cur.wait_stream(self.comm_stream)
        world, rank = self.comm.world, self.comm.rank
        if world > 1:
            self.comm.barrier(stream=cur)
        with torch.no_grad():
            for b in self.buckets:
                shard = b.numel // world
                src = shard_of(b).to(self.dtype)
                mine = b.param[rank * shard:(rank + 1) * shard]
                for peer in range(world):
                    (mine if peer == rank else self.comm.peer_tensor(mine, peer)).copy_(src)
        if world > 1:
            self.comm.barrier(stream=cur)

    def _adamw_hp(self, step: int) -> list:
        return [self.lr, self.betas[0], self.betas[1], self.eps, self.weight_decay, self._grad_scale, float(step), 0.0]

    def _state(self, b: _Bucket) -> tuple:
        """The fp32 tensors the fused kernel updates for bucket `b`, master first."""
        return b.state

    @property
    def micro_step(self) -> int:
        """The micro-batch of the current optimizer step that the next backward belongs to (0..accumulation_steps-1)."""
        return self._micro

    @property
    def kernel_launches(self) -> int:
        return self.comm.launches

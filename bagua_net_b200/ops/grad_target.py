"""Where a parameter's gradient should be WRITTEN: a registry between the training engine and the gradient producers.

``BnetDDP`` keeps every gradient in one flat buffer that its fused all-reduce + optimizer kernels read.  Autograd normally
produces a gradient in a tensor of its own and then accumulates it into ``p.grad`` (an add: three passes over the parameter's
bytes), or — when ``p.grad`` is ``None`` — adopts the produced tensor as it is.  The engine therefore leaves ``p.grad = None``
before a backward pass and registers, per parameter, the slice of the flat buffer its gradient belongs in.  A producer that can
write its result anywhere (a GEMM with an output argument, our own kernels) asks ``lookup(weight)`` and, if it gets a slice of
matching shape / dtype / layout, writes there and returns ``adopt(slice)`` — a fresh tensor object over the same memory, which
autograd adopts without touching the data.  Everything else keeps working unchanged: the engine's hook copies a gradient that
arrived in a tensor of its own into the slice (two passes instead of the add's three).

The reference has no training engine (SURVEY.md section 2.5: data parallelism is its consumer); this belongs to the GPU side."""
from __future__ import annotations

import weakref

import torch

# data_ptr of the parameter (its slice of the flat parameter buffer) -> [gradient slice, weak reference to the engine that owns
# both buffers (or None), claimed].  An entry whose engine is gone is dropped at the next lookup: its memory may have been
# unmapped, and a new tensor could reuse the address.  `claimed`: a slice is handed out ONCE per backward pass — a parameter
# used twice in the graph (weight sharing) gets its second gradient in a tensor of its own, which autograd then adds to the
# adopted slice, as it should; the engine's hook releases the claim when the parameter's gradient is complete.
_TARGETS: dict[int, list] = {}


def register(param: torch.Tensor, grad_slice: torch.Tensor, owner=None) -> None:
    _TARGETS[param.data_ptr()] = [grad_slice, weakref.ref(owner) if owner is not None else None, False]


def release(param: torch.Tensor) -> None:
    e = _TARGETS.get(param.data_ptr())
    if e is not None:
        e[2] = False


def unregister(param: torch.Tensor) -> None:
    _TARGETS.pop(param.data_ptr(), None)


def lookup(weight: torch.Tensor, shape=None, dtype=None) -> torch.Tensor | None:
    """The registered gradient slice of `weight` if it can take a result of `shape` / `dtype` (default: the weight's own) with
    the weight's strides and 16-byte alignment; None otherwise (the caller then allocates as usual)."""
    entry = _TARGETS.get(weight.data_ptr())
    if entry is None:
        return None
    t, owner, claimed = entry
    if owner is not None and owner() is None:
        del _TARGETS[weight.data_ptr()]
        return None
    if claimed:
        return None
    if tuple(t.shape) != tuple(shape if shape is not None else weight.shape) or t.dtype != (dtype or weight.dtype):
        return None
    if t.stride() != weight.stride() or t.data_ptr() % 16 or t.device != weight.device:
        return None
    entry[2] = True
    return t


def adopt(grad_slice: torch.Tensor) -> torch.Tensor:
    """What a producer returns after writing into `grad_slice`: a new tensor object over the same memory (autograd adopts a
    gradient it holds the only reference to; the registry keeps its own reference to the slice itself)."""
    return grad_slice.detach()

"""What the CPU tests of BnetDDP's host logic put in place of the GPU: a comm that does every SymmComm call the engine
makes with the same arithmetic in plain PyTorch (one rank, host memory), stubs for the CUDA stream / event calls (the
`cpu_engine` fixture) and a small model.  bagua_net_b200/parallel/ddp.py itself runs unmodified.  Also the torch side
the engine is trained against: the hyper-parameters, an engine / torch.optim pair, the batches and the reference step."""
import contextlib
import math

import pytest
import torch

from bagua_net_b200.parallel.comm import CLIP_ROW, LARS_CHUNK, check_group_segments, check_lars_segments, check_lars_tensors
from bagua_net_b200.parallel.ddp import BnetDDP


class FakeStream:
    def wait_event(self, ev):
        pass

    def wait_stream(self, s):
        pass

    def synchronize(self):
        pass


class FakeEvent:
    def record(self, s=None):
        pass


class FakeComm:
    """What BnetDDP needs from SymmComm, for one rank, in host memory.  The methods take SymmComm's parameters and
    assert the argument contracts that SymmComm enforces on the engine's calls.  `log` lists every call in order as
    (kind, size):

    sgd / adamw / sgd_groups / adamw_groups (one-kernel step) and norm / accum (stage 1): the gradient numel;  coef: the
    number of partial rows;  barrier: None;  apply / apply_groups (stage-3 SGD / AdamW) and lars_apply: the param numel;
    lars_norm and ema_update: the master numel;  lars_trust: the number of tensors;  ema_advance: None."""

    def __init__(self):
        self.world, self.rank, self.launches = 1, 0, 0
        self.log = []
        self.steps_seen = []               # the step count every AdamW update read
        self.coef_scales = []              # the gradient scale of every coefficient launch
        self.apply_scales = []             # ... and of every SGD / AdamW update from the scratch
        self._lars_nslots = {}             # id of a segment table from lars_segments -> (the table, its norm slots)
        self._group_tables = {}            # id of a segment table from group_segments -> (shard vectors, groups)

    def _launched(self, kind, size):
        self.launches += 1
        self.log.append((kind, size))

    def alloc(self, numel, dtype, align=256):
        return torch.zeros(numel, dtype=dtype)

    def all_reduce(self, t, op="sum", algo="auto", channel=1, nblocks=0, stream=None):
        return t

    def barrier(self, channel=2, stream=None):
        assert channel == 0
        self.log.append(("barrier", None))       # (no kernel on one rank, as SymmComm.barrier)

    # ------------------------------------------------------------------ the optimizer updates, from a summed gradient
    def _sgd(self, g, param, master, mom, lr, momentum, weight_decay, grad_scale, hp):
        """Returns the gradient scale it used."""
        if hp is not None:
            lr, momentum, weight_decay, grad_scale = (float(v) for v in hp[:4])
        elif grad_scale is None:
            grad_scale = 1.0 / self.world
        g = g.float() * grad_scale + weight_decay * master        # mean gradient + L2 term on the fp32 master weights
        mom.mul_(momentum).add_(g)
        master.sub_(lr * mom)
        param.copy_(master.to(param.dtype))
        return grad_scale

    def _adamw(self, g, param, master, exp_avg, exp_avg_sq, hp):
        """Returns the gradient scale it used."""
        assert hp.dtype == torch.float32 and hp.numel() == 8
        lr, b1, b2, eps, wd, scale, step = (float(v) for v in hp[:7])
        t = step + 1
        g = g.float() * scale
        master.mul_(1 - lr * wd)
        exp_avg.mul_(b1).add_(g, alpha=1 - b1)
        exp_avg_sq.mul_(b2).addcmul_(g, g, value=1 - b2)
        denom = (exp_avg_sq.sqrt() / math.sqrt(1 - b2 ** t)).add_(eps)
        master.addcdiv_(exp_avg, denom, value=-lr / (1 - b1 ** t))
        param.copy_(master.to(param.dtype))
        self.steps_seen.append(step)
        return scale

    # ------------------------------------------------------------------ the one-kernel step
    def fused_allreduce_sgd(self, grad, param, master, mom, lr, momentum, weight_decay, grad_scale=None, zero_grads=True, channel=0,
                            nblocks=0, stream=None, hp=None):
        self._sgd(grad, param, master, mom, lr, momentum, weight_decay, grad_scale, hp)
        if zero_grads:
            grad.zero_()
        self._launched("sgd", grad.numel())

    def fused_allreduce_adamw(self, grad, param, master, exp_avg, exp_avg_sq, hp, zero_grads=True, channel=0, nblocks=0,
                              stream=None):
        self._adamw(grad, param, master, exp_avg, exp_avg_sq, hp)
        if zero_grads:
            grad.zero_()
        self._launched("adamw", grad.numel())

    # ------------------------------------------------------------------ the staged step: stage 1, coefficient, apply
    def _stage1(self, kind, grad, scratch, partial, add):
        assert scratch.dtype == torch.float32 and scratch.numel() * self.world == grad.numel()
        assert partial.dtype == torch.float64 and partial.numel() == CLIP_ROW
        if add:
            scratch.add_(grad.float())
        else:
            scratch.copy_(grad.float())
        partial.zero_()
        partial[0] = scratch.double().square().sum()         # over the (new) scratch values
        grad.zero_()
        self._launched(kind, grad.numel())

    def fused_clip_reduce_norm(self, grad, scratch, partial, channel=0, nblocks=0, stream=None):
        self._stage1("norm", grad, scratch, partial, add=False)

    def fused_accum_reduce_norm(self, grad, scratch, partial, channel=0, nblocks=0, stream=None):
        self._stage1("accum", grad, scratch, partial, add=True)

    def fused_clip_coef(self, partials, xchg, clip, grad_scale=None, channel=0, stream=None):
        assert partials.shape[1] == CLIP_ROW and xchg.numel() >= self.world and clip.numel() == 4
        gs = 1.0 / self.world if grad_scale is None else grad_scale
        self.coef_scales.append(gs)
        total = torch.tensor(math.sqrt(float(partials.sum())) * gs, dtype=torch.float32)
        clip[1] = total
        clip[2] = torch.clamp(clip[0] / (total + 1e-6), max=1.0)
        self._launched("coef", partials.shape[0])

    def fused_clip_apply_sgd(self, param, scratch, clip, master, mom, lr, momentum, weight_decay, grad_scale=None, channel=0,
                             nblocks=0, stream=None, hp=None):
        self.apply_scales.append(self._sgd(scratch * clip[2], param, master, mom, lr, momentum, weight_decay, grad_scale, hp))
        self._launched("apply", param.numel())

    def fused_clip_apply_adamw(self, param, scratch, clip, master, exp_avg, exp_avg_sq, hp, channel=0, nblocks=0, stream=None):
        self.apply_scales.append(self._adamw(scratch * clip[2], param, master, exp_avg, exp_avg_sq, hp))
        self._launched("apply", param.numel())

    # ------------------------------------------------------------------ parameter groups: each segment of the validated
    # table updated with its group's row
    def group_segments(self, table, shard_vecs, ngroups):
        check_group_segments(table, shard_vecs, ngroups)
        t = torch.tensor(table, dtype=torch.int32).reshape(-1, 4)
        self._group_tables[id(t)] = (shard_vecs, ngroups)
        return t

    def _per_segment(self, param, segs, groups, hp, update):
        shard_vecs, ngroups = self._group_tables[id(segs)]
        e = 16 // param.element_size()
        assert shard_vecs * e == param.numel() and groups.shape == (groups.shape[0], 4) and groups.shape[0] >= ngroups
        for vec0, nvec, g, _ in segs.tolist():
            h = hp.clone()
            h[0], h[4 if hp.numel() == 8 else 2] = groups[g, 0], groups[g, 1]
            update(slice(vec0 * e, (vec0 + nvec) * e), h)

    def _sgd_groups(self, g, param, master, mom, hp, groups, segs):
        assert hp.numel() == 4
        self._per_segment(param, segs, groups, hp, lambda s, h: self._sgd(g[s], param[s], master[s], mom[s], 0, 0, 0, None, h))
        return float(hp[3])

    def _adamw_groups(self, g, param, master, exp_avg, exp_avg_sq, hp, groups, segs):
        steps = len(self.steps_seen)
        self._per_segment(param, segs, groups, hp,
                          lambda s, h: self._adamw(g[s], param[s], master[s], exp_avg[s], exp_avg_sq[s], h))
        del self.steps_seen[steps + 1:]    # (one step, however many segments)
        return float(hp[5])

    def fused_allreduce_sgd_groups(self, grad, param, master, mom, hp, groups, segs, zero_grads=True, channel=0, nblocks=0,
                                   stream=None):
        self._sgd_groups(grad, param, master, mom, hp, groups, segs)
        grad.zero_()
        self._launched("sgd_groups", grad.numel())

    def fused_allreduce_adamw_groups(self, grad, param, master, exp_avg, exp_avg_sq, hp, groups, segs, zero_grads=True,
                                     channel=0, nblocks=0, stream=None):
        self._adamw_groups(grad, param, master, exp_avg, exp_avg_sq, hp, groups, segs)
        grad.zero_()
        self._launched("adamw_groups", grad.numel())

    def fused_clip_apply_sgd_groups(self, param, scratch, clip, master, mom, hp, groups, segs, channel=0, nblocks=0,
                                    stream=None):
        self.apply_scales.append(self._sgd_groups(scratch * clip[2], param, master, mom, hp, groups, segs))
        self._launched("apply_groups", param.numel())

    def fused_clip_apply_adamw_groups(self, param, scratch, clip, master, exp_avg, exp_avg_sq, hp, groups, segs, channel=0,
                                      nblocks=0, stream=None):
        self.apply_scales.append(self._adamw_groups(scratch * clip[2], param, master, exp_avg, exp_avg_sq, hp, groups, segs))
        self._launched("apply_groups", param.numel())

    # ------------------------------------------------------------------ LARS: norm, trust, apply
    def lars_segments(self, table, shard_vecs, ntensors):
        t = torch.tensor(table, dtype=torch.int32).reshape(-1, 4)
        self._lars_nslots[id(t)] = (t, check_lars_segments(table, shard_vecs, ntensors))
        return t

    def lars_tensors(self, table, nslots):
        check_lars_tensors(table, nslots)
        return torch.tensor(table, dtype=torch.int32).reshape(-1, 4)

    def fused_lars_norm(self, master, scratch, segs, slots, dtype, nblocks=0, stream=None):
        table, nslots = self._lars_nslots[id(segs)]
        assert table is segs and slots.shape == (nslots, 2)
        e = 16 // torch.empty((), dtype=dtype).element_size()
        for vec0, nvec, _, slot0 in segs.tolist():
            for c in range((nvec + LARS_CHUNK - 1) // LARS_CHUNK):
                a, b = (vec0 + c * LARS_CHUNK) * e, (vec0 + min(nvec, (c + 1) * LARS_CHUNK)) * e
                slots[slot0 + c] = torch.stack([master[a:b].double().square().sum(), scratch[a:b].double().square().sum()])
        self._launched("lars_norm", master.numel())

    def fused_lars_trust(self, slots, tensors, xchg, clip, hp, scal, trust, channel=0, stream=None):
        assert xchg.numel() >= 2 * self.world * tensors.shape[0]
        f = lambda v: torch.tensor(float(v), dtype=torch.float32)  # noqa: E731
        gscale, wd, eta, eps, coef = f(hp[3]), f(hp[2]), f(hp[4]), f(hp[5]), f(clip[2])
        for j, (slot0, n, excluded, _) in enumerate(tensors.tolist()):
            w2, g2 = (float(v) for v in slots[slot0:slot0 + n].sum(0)) if n else (0.0, 0.0)
            wn, gn = f(math.sqrt(w2)), f(math.sqrt(g2) * float(gscale) * float(coef))
            live = not excluded and wn != 0 and gn != 0
            t = eta * wn / (gn + wd * wn + eps) if live else torch.tensor(1.0)
            scal[j, 0], scal[j, 1], trust[j] = gscale * coef * t, wd * t if live else 0.0, t
        self._launched("lars_trust", tensors.shape[0])

    def fused_lars_apply(self, param, scratch, segs, scal, hp, master, mom, channel=0, nblocks=0, stream=None):
        lr, mu = float(hp[0]), float(hp[1])
        e = 16 // param.element_size()
        for vec0, nvec, tensor, _ in segs.tolist():
            s = slice(vec0 * e, (vec0 + nvec) * e)
            mom[s].mul_(mu).add_(scratch[s] * scal[tensor, 0] + scal[tensor, 1] * master[s])
            master[s].sub_(lr * mom[s])
        param.copy_(master.to(param.dtype))
        self._launched("lars_apply", param.numel())

    # ------------------------------------------------------------------ the EMA kernels: the gate of optim::ema_gate on
    # the block {1 - decay, every, step, n_averaged}, torch.lerp
    def ema_update(self, master, ema, blk, nblocks=0, stream=None):
        assert blk.dtype == torch.float32 and blk.numel() == 4 and ema.shape == master.shape
        w, every, step, n = blk.tolist()
        if (int(step) + 1) % int(every) == 0:
            ema.copy_(master if n == 0 else torch.lerp(ema, master, w))
        self._launched("ema_update", master.numel())

    def ema_advance(self, blk, stream=None):
        assert blk.dtype == torch.float32 and blk.numel() == 4
        w, every, step, n = blk.tolist()
        if (int(step) + 1) % int(every) == 0:
            blk[3] += 1
        blk[2] += 1
        self._launched("ema_advance", None)


@pytest.fixture
def cpu_engine(monkeypatch):
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "Event", lambda *a, **k: FakeEvent())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: FakeStream())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "stream", lambda s: contextlib.nullcontext())
    return monkeypatch


def small_model(channels_last=True):
    torch.manual_seed(3)
    m = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.ReLU(), torch.nn.Conv2d(8, 8, 3, padding=1), torch.nn.ReLU(),
                            torch.nn.AdaptiveAvgPool2d(2), torch.nn.Flatten(), torch.nn.Linear(32, 10))
    return m.to(memory_format=torch.channels_last) if channels_last else m


class Branchy(torch.nn.Module):
    """small_model plus layers that fill a bucket each, registered first: `unused` never gets a gradient, `late` (built
    when asked) only while `use_late` is on."""

    def __init__(self, channels_last=True, late=False):
        super().__init__()
        torch.manual_seed(4)
        self.unused = torch.nn.Linear(32, 32, bias=False)
        if late:
            self.late = torch.nn.Linear(32, 32, bias=False)
        self.net = small_model(channels_last)
        self.use_late = False

    def forward(self, x):
        h = self.net[:-1](x)
        if self.use_late:
            h = h + self.late(h)
        return self.net[-1](h)


# ------------------------------------------------------------------ the torch side
LARC = dict(weight_decay=5e-4, trust_coefficient=0.02, eps=1e-8)
HYPER = {"sgd": dict(lr=0.05, momentum=0.9, weight_decay=1e-3),
         "adamw": dict(lr=3e-3, betas=(0.85, 0.99), eps=1e-7, weight_decay=0.05),
         "lars": dict(lr=0.5, momentum=0.9, **LARC)}


def make_pair(optimizer, model=small_model, channels_last=True, dtype=torch.float64, **engine_kw):
    """(torch reference in `dtype`, its torch.optim optimizer, the engine's model, the engine with ~2 KB buckets): both
    from `model(channels_last)` and HYPER[optimizer].  LARS's reference optimizer is SGD without weight decay: larc_
    applies it."""
    ref, net = model(channels_last).to(dtype), model(channels_last)
    h = HYPER[optimizer]
    if optimizer == "adamw":
        opt = torch.optim.AdamW(ref.parameters(), **h)
    else:
        opt = torch.optim.SGD(ref.parameters(), lr=h["lr"], momentum=h["momentum"],
                              weight_decay=0.0 if optimizer == "lars" else h["weight_decay"])
    eng = BnetDDP(net, optimizer=optimizer, bucket_mb=0.002, comm=FakeComm(), **h, **engine_kw)
    return ref, opt, net, eng


def batch(step, n, seed, channels_last=True):
    torch.manual_seed(seed + step)
    x, y = torch.randn(n, 3, 8, 8), torch.randint(0, 10, (n,))
    return (x.contiguous(memory_format=torch.channels_last) if channels_last else x), y


def larc_(params, weight_decay, trust_coefficient, eps):
    """NVIDIA Apex LARC(clip=False) on the .grad of `params`: weight decay and the trust ratio folded into the gradient
    of every tensor of more than one dimension that has one."""
    with torch.no_grad():
        for p in params:
            if p.grad is None or p.dim() <= 1:
                continue
            wn, gn = p.norm(), p.grad.norm()
            if wn != 0 and gn != 0:
                t = trust_coefficient * wn / (gn + wn * weight_decay + eps)
                p.grad.add_(p, alpha=weight_decay).mul_(t)


def torch_step(ref, opt, x, y, k=1, max_norm=None, lars=None) -> float:
    """One optimizer step of the torch reference on the batch: k equal micro-batches accumulated as loss / k each,
    clip_grad_norm_ to `max_norm` (None: inf, which multiplies the gradients by exactly 1), Apex LARC with
    `lars` = dict(weight_decay, trust_coefficient, eps), then `opt`.  Returns the pre-clip gradient norm."""
    opt.zero_grad()
    dtype = next(ref.parameters()).dtype
    for xs, ys in zip(x.chunk(k), y.chunk(k)):
        (torch.nn.functional.cross_entropy(ref(xs.to(dtype)), ys) / k).backward()
    norm = torch.nn.utils.clip_grad_norm_(ref.parameters(), math.inf if max_norm is None else max_norm)
    if lars is not None:
        larc_(ref.parameters(), **lars)
    opt.step()
    return float(norm)


def close_params(net, ref, atol, tag=None, rtol=0.0):
    for a, b in zip(net.parameters(), ref.parameters()):
        assert torch.allclose(a.to(b.dtype), b, rtol=rtol, atol=atol), (tag, float((a.to(b.dtype) - b).abs().max()))

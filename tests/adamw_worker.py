"""Per-rank bodies of the fused AdamW GPU tests (launched by tests/test_fused_adamw.py, one process per GPU)."""
from __future__ import annotations

import math
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

RANK = int(os.environ.get("RANK", "0"))
WORLD = int(os.environ.get("WORLD_SIZE", "1"))
LOCAL = int(os.environ.get("LOCAL_RANK", "0"))

U = 2.0 ** -24                 # fp32 unit roundoff
FLOOR = 4 * 2.0 ** -149        # results in the subnormal range round to a multiple of 2^-149
STEP = 6                       # index of the step count in the hyper-parameter block


def setup():
    torch.cuda.set_device(LOCAL)
    if WORLD > 1:
        dist.init_process_group("nccl")


def teardown():
    if WORLD > 1 and dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()


def f32(x):
    """A hyper-parameter as the kernel sees it (rounded to fp32), in double."""
    return float(torch.tensor(x, dtype=torch.float32))


def same_on_every_rank(t: torch.Tensor) -> bool:
    if WORLD == 1:
        return True
    lst = [torch.empty_like(t) for _ in range(WORLD)]
    dist.all_gather(lst, t.contiguous())
    return all(torch.equal(lst[0].view(torch.uint8), x.view(torch.uint8)) for x in lst)


# ------------------------------------------------------------------ float64 AdamW with an fp32 error bound
def adamw_f64(p, m, v, g, hp):
    """One AdamW step in float64 on the kernel's fp32 inputs, and the error the kernel's fp32 arithmetic may add in this
    step (the per-operation rounding analysis of csrc/tests/optim_emu_test.cc).  Returns the new (p, m, v) and, per
    element, (local bound of m, v, p) together with the derivatives the caller needs to carry earlier steps' errors."""
    lr, b1, b2, eps, wd, gs, step = (f32(x) for x in hp[:7])
    t = step + 1
    g = g * gs
    M = b1 * m.abs() + (1 - b1) * g.abs()
    V = b2 * v + (1 - b2) * g * g
    m1 = b1 * m + (1 - b1) * g
    v1 = V
    S = lr / (1 - b1 ** t)
    bc2s = (1 - b2 ** t) ** 0.5
    D = v1.sqrt() / bc2s + eps
    decay = 1 - lr * wd
    p2 = p * decay - S * m1 / D
    return p2, m1, v1, dict(M=M, m1=m1, v1=v1, S=S, D=D, bc2s=bc2s, decay=decay, b1=b1, b2=b2, p=p, p2=p2)


class Reference:
    """float64 AdamW over several steps, with the element-wise bound |kernel - reference| <= B that fp32 rounding in every
    step allows, errors of earlier steps carried forward: B_m' = b1 B_m + 4u M, B_v' = b2 B_v + 6u V,
    B_p' = (1 - lr wd) B_p + 3u|p| + 2u|p'| + S/D (B_m' + 5u M + 10u|m'|) + S|m'|/D * (dsqrt(B_v')/(bc2 D) + 7u)."""

    def __init__(self, p0: torch.Tensor):
        self.p = p0.double()
        self.m = torch.zeros_like(self.p)
        self.v = torch.zeros_like(self.p)
        self.bp = torch.zeros_like(self.p)
        self.bm = torch.zeros_like(self.p)
        self.bv = torch.zeros_like(self.p)

    def step(self, g: torch.Tensor, hp):
        p2, m1, v1, k = adamw_f64(self.p, self.m, self.v, g.double(), hp)
        self.bm = k["b1"] * self.bm + 4 * U * k["M"] + FLOOR
        self.bv = k["b2"] * self.bv + 6 * U * v1 + FLOOR
        sq = v1.sqrt()
        dsq = torch.minimum(self.bv / (2 * sq).clamp_min(1e-300), self.bv.sqrt())
        rel_d = dsq / k["bc2s"] / k["D"] + 7 * U
        s_d = k["S"] / k["D"]
        bupd = s_d * (self.bm + 5 * U * k["M"] + 10 * U * m1.abs()) + s_d * m1.abs() * rel_d
        self.bp = k["decay"] * self.bp + 3 * U * self.p.abs() + 2 * U * p2.abs() + bupd + FLOOR
        self.p, self.m, self.v = p2, m1, v1

    def worst(self, master, exp_avg, exp_avg_sq):
        """Largest error/bound ratio of the three fp32 tensors."""
        r = 0.0
        for got, want, b in ((master, self.p, self.bp), (exp_avg, self.m, self.bm), (exp_avg_sq, self.v, self.bv)):
            # (a NaN or infinite result where the reference is finite counts as outside the bound: torch's max() of a
            # tensor with a NaN is NaN, and Python's max(r, nan) would drop it)
            r = max(r, float(((got.double() - want).abs() / b).nan_to_num(nan=math.inf, posinf=math.inf).max()))
        return r


# ------------------------------------------------------------------ the kernel against float64
def grads_for(step, n, dtype, scale=1.0):
    """Every rank's gradient of `step`: multiples of 2^-q in [-1, 1] with q = 6 up to four ranks and
    q = 8 - ceil(log2 WORLD) above, so that every partial sum over the ranks is a multiple of 2^-q of magnitude at most
    WORLD * 2^q <= 2^8: exact in bf16 (8 significant bits) and fp32 whichever way and in whatever order the kernel reduces
    (in the switch, which rounds its sum to bf16, with peer loads in fp32, or locally).  With q = 6 at eight ranks a sum
    could reach 512 and need 9 bits; up to four ranks the data is the same as with q = 6 everywhere."""
    q = 64 if WORLD <= 4 else 2 ** (8 - math.ceil(math.log2(WORLD)))
    gs = []
    for r in range(WORLD):
        gen = torch.Generator(device="cuda").manual_seed(1000 * step + r)
        gs.append((torch.randint(-q, q + 1, (n,), device="cuda", generator=gen).float() / q * scale).to(dtype))
    return gs


def job_kernel():
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(256 << 20)
    for dtype in (torch.bfloat16, torch.float32):
        n = 8 * WORLD * 4099                      # per-rank vectors leave a tail for every grid size below
        shard = n // WORLD
        guard = 16 * WORLD * 8                    # guard elements on both sides of param and grad (16-byte aligned)
        sentinel = 3.0
        pbuf, gbuf = comm.alloc(n + 2 * guard, dtype), comm.alloc(n + 2 * guard, dtype)
        param, grad = pbuf[guard:guard + n], gbuf[guard:guard + n]
        torch.manual_seed(7)
        p0 = (torch.randn(n, device="cuda") * 0.5).to(dtype)
        lrs = [1e-2, 1e-2, 3e-3, 3e-3, 1e-3]       # the learning rate changes between steps
        hp = torch.zeros(8, device="cuda", dtype=torch.float32)

        def run(nblocks, step0=0, nsteps=5, specials=None):
            pbuf.fill_(sentinel)
            gbuf.fill_(sentinel)
            param.copy_(p0)
            master = param[RANK * shard:(RANK + 1) * shard].float().contiguous()
            exp_avg, exp_avg_sq = torch.zeros_like(master), torch.zeros_like(master)
            for s in range(nsteps):
                hp.copy_(torch.tensor([lrs[s], 0.9, 0.999, 1e-8, 0.01, 1.0 / WORLD, step0 + s, 0.0]))
                g = grads_for(s, n, dtype)[RANK]
                if specials is not None:
                    g = g.clone()
                    g[specials[0]] = specials[1].to(dtype)
                grad.copy_(g)
                torch.cuda.synchronize()
                if WORLD > 1:
                    dist.barrier()
                comm.fused_allreduce_adamw(grad, param, master, exp_avg, exp_avg_sq, hp, nblocks=nblocks)
                torch.cuda.synchronize()
                assert int((grad != 0).sum()) == 0, "gradients were not re-zeroed"
                for buf in (pbuf, gbuf):
                    assert bool((buf[:guard] == sentinel).all() and (buf[guard + n:] == sentinel).all()), "guard overwritten"
            return param.clone(), master, exp_avg, exp_avg_sq

        # 5 steps, learning-rate changes, against float64
        got = run(0)
        ref = Reference(p0.float()[RANK * shard:(RANK + 1) * shard])
        for s in range(5):
            gsum = torch.stack([x.double() for x in grads_for(s, n, dtype)]).sum(0)[RANK * shard:(RANK + 1) * shard]
            ref.step(gsum, [lrs[s], 0.9, 0.999, 1e-8, 0.01, 1.0 / WORLD, s])
        w = ref.worst(*got[1:])
        assert w <= 1.0, f"{dtype}: kernel outside the fp32 bound of float64 AdamW (worst error/bound {w:.3f})"
        mine = got[0][RANK * shard:(RANK + 1) * shard]
        assert torch.equal(mine.view(torch.uint8), got[1].to(dtype).view(torch.uint8)), "parameters != master.to(dtype)"
        assert same_on_every_rank(got[0]), "ranks hold different parameters"
        # the same bits for every grid size
        for nb in (1, 7, 132, 264):
            other = run(nb)
            for a, b in zip(got, other):
                assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f"{dtype}: nblocks={nb} changes the result"
        # a late step: the bias corrections at t = 10^5 + 1, 10^5 + 2
        late = run(0, step0=100000 - 1, nsteps=2)
        ref_l = Reference(p0.float()[RANK * shard:(RANK + 1) * shard])
        for s in range(2):
            gsum = torch.stack([x.double() for x in grads_for(s, n, dtype)]).sum(0)[RANK * shard:(RANK + 1) * shard]
            ref_l.step(gsum, [lrs[s], 0.9, 0.999, 1e-8, 0.01, 1.0 / WORLD, 100000 - 1 + s])
        wl = ref_l.worst(*late[1:])
        assert wl <= 1.0, f"{dtype}: step 10^5 outside the bound (worst error/bound {wl:.3f})"
        # NaN / +-Inf gradient elements: the NaN and Inf pattern of torch.optim.AdamW with its default implementation
        # (step 1 from zero state)
        idx = torch.arange(0, n, 37, device="cuda")
        vals = torch.tensor([float("nan"), float("inf"), float("-inf")], device="cuda").repeat(len(idx) // 3 + 1)[:len(idx)]
        bad = run(0, nsteps=1, specials=(idx, vals))
        gsum = torch.stack([x.float() for x in grads_for(0, n, dtype)]).sum(0)
        gsum[idx] = vals * WORLD                  # (every rank puts the specials at the same elements)
        tp = torch.nn.Parameter(p0.float().clone())
        opt = torch.optim.AdamW([tp], lr=lrs[0], betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01)
        tp.grad = gsum / WORLD
        opt.step()
        st = opt.state[tp]
        for name, a, b in (("master", bad[1], tp.detach()), ("exp_avg", bad[2], st["exp_avg"]),
                           ("exp_avg_sq", bad[3], st["exp_avg_sq"])):
            b = b[RANK * shard:(RANK + 1) * shard]
            assert torch.equal(a.isnan(), b.isnan()), f"{dtype}: NaN pattern of {name} differs from torch"
            assert torch.equal(a.isinf(), b.isinf()), f"{dtype}: Inf pattern of {name} differs from torch"
            assert torch.equal(a[b.isinf()], b[b.isinf()]), f"{dtype}: the signs of {name}'s infinities differ from torch"
        assert int(bad[1].isnan().sum()) == len(idx[(idx >= RANK * shard) & (idx < (RANK + 1) * shard)])
        print(f"rank {RANK}: fused adamw {dtype} ok: worst error/bound {w:.3f} (5 steps), {wl:.3f} (step 1e5); "
              f"bitwise equal for nblocks 1/7/132/264; NaN pattern = torch (multicast={comm.has_multicast})", flush=True)
    assert comm.status() == 0
    teardown()


def job_staggered():
    """The race of the CTA-paired gradient zeroing, redone for AdamW: 64 CTAs on a side stream under a concurrent GEMM.
    Integer gradients and beta1 = beta2 = 0: exp_avg must equal the mean gradient bitwise, so a lost or doubled
    contribution shows."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(512 << 20)
    n = 8 * WORLD * (64 * 512 * 5 + 4099)          # per-rank vectors: NOT a multiple of 64 blocks x 512 threads
    dtype = torch.bfloat16
    param, grad = comm.alloc(n, dtype), comm.alloc(n, dtype)
    shard = n // WORLD
    master = torch.zeros(shard, device="cuda", dtype=torch.float32)
    exp_avg, exp_avg_sq = torch.zeros_like(master), torch.zeros_like(master)
    hp = torch.tensor([1.0, 0.0, 0.0, 1.0, 0.0, 1.0 / WORLD, 0.0, 0.0], device="cuda")
    side = torch.cuda.Stream()
    a = torch.randn(8192, 8192, device="cuda", dtype=torch.bfloat16)
    for step in range(6):
        grad.copy_(((torch.arange(n, device="cuda") * 3 + RANK + step) % 5 - 2).to(dtype))
        param.zero_()
        master.zero_()
        exp_avg.zero_()
        exp_avg_sq.zero_()
        torch.cuda.synchronize()
        if WORLD > 1:
            dist.barrier()
        for _ in range(3):
            a @ a                                   # fills every SM while the fused kernel's CTAs trickle in
        with torch.cuda.stream(side):
            comm.fused_allreduce_adamw(grad, param, master, exp_avg, exp_avg_sq, hp, zero_grads=True, nblocks=64, stream=side)
        torch.cuda.synchronize()
        want = (sum(((torch.arange(n, device="cuda") * 3 + r + step) % 5 - 2).float() for r in range(WORLD)) / WORLD)
        bad = int((exp_avg != want[RANK * shard:(RANK + 1) * shard]).sum())
        assert bad == 0, f"rank {RANK} step {step}: {bad} wrong elements (staggered CTAs corrupted the reduction)"
        assert torch.equal(exp_avg_sq, exp_avg * exp_avg), "exp_avg_sq != g^2"
        assert int((grad != 0).sum()) == 0, "gradients were not re-zeroed"
    assert comm.status() == 0
    print(f"rank {RANK}: fused adamw with 64 staggered CTAs under a concurrent GEMM ok (world {WORLD})", flush=True)
    teardown()


# ------------------------------------------------------------------ the engine against torch.optim.AdamW
KW = dict(width_div=8, fc_dim=128, image_size=32, num_classes=10, dropout=0.0)
HYPER = dict(lr=2e-3, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.05)


def batch(step):
    xs, ys = [], []
    for r in range(WORLD):
        torch.manual_seed(1000 + 10 * step + r)
        xs.append(torch.randn(4, 3, 32, 32, device="cuda"))
        ys.append(torch.randint(0, 10, (4,), device="cuda"))
    return xs, ys


def lr_at(step):
    return HYPER["lr"] * (0.5 if step >= 4 else 1.0)        # a schedule change after step 4


def make_engine(graph, model=None):
    from bagua_net_b200.models import build_model
    from bagua_net_b200.parallel import BnetDDP

    if model is None:
        torch.manual_seed(0)
        model = build_model("vgg16", **KW).cuda()
    model = model.to(memory_format=torch.channels_last)
    eng = BnetDDP(model, bucket_mb=0.25, optimizer="adamw", **HYPER)
    eng.enable_cuda_graph(graph)
    return model, eng


def engine_step(eng, step):
    xs, ys = batch(step)
    eng.set_lr(lr_at(step))
    return eng.train_step(xs[RANK].contiguous(memory_format=torch.channels_last), ys[RANK])


def job_engine():
    from bagua_net_b200.models import build_model

    setup()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    for graph in (False, True):
        torch.manual_seed(0)
        ref = build_model("vgg16", **KW).cuda()
        model, eng = make_engine(graph)
        assert len(eng.buckets) > 1
        p0 = [p.detach().clone() for p in ref.parameters()]
        opt = torch.optim.AdamW(ref.parameters(), **HYPER)
        assert float(eng._hp[STEP]) == 0.0
        g = None
        snap = None
        for step in range(6):
            engine_step(eng, step)
            if graph:
                if g is None:
                    g = eng._graph
                assert eng._graph is g, "the graph was re-captured (learning-rate change or step count)"
            torch.cuda.synchronize()
            # the capture's warm-up steps are undone and the capture itself runs nothing: one advance per step
            assert float(eng._hp[STEP]) == step + 1, (step, float(eng._hp[STEP]))
            xs, ys = batch(step)
            for grp in opt.param_groups:
                grp["lr"] = lr_at(step)
            opt.zero_grad()
            torch.nn.functional.cross_entropy(ref(torch.cat(xs)), torch.cat(ys)).backward()
            opt.step()
            if step == 2:
                snap = ({k: v.clone() for k, v in model.state_dict().items()}, eng.optimizer_state_dict())
        torch.cuda.synchronize()
        num, den, worst = 0.0, 0.0, 0.0
        for a, b, s in zip(model.parameters(), ref.parameters(), p0):
            du, dr = (a.detach().double() - s.double()), (b.detach().double() - s.double())
            e, r = float((du - dr).norm()), float(dr.norm())
            num, den = num + e * e, den + r * r
            worst = max(worst, e / r if r > 0 else (0.0 if e == 0 else float("inf")))
        total = (num / den) ** 0.5
        assert total < 1e-3 and worst < 1e-2, f"graph={graph}: updates differ from torch AdamW: total {total:.2e}, worst {worst:.2e}"
        assert same_on_every_rank(eng.flat_param), "ranks hold different parameters"
        # checkpoint after step 3, resumed into a fresh engine: the same bits at step 6
        torch.manual_seed(0)
        fresh = build_model("vgg16", **KW).cuda()
        fresh.load_state_dict(snap[0])
        fm, fe = make_engine(graph, fresh)
        fe.load_optimizer_state_dict(snap[1])
        assert float(fe._hp[STEP]) == 3.0
        for step in range(3, 6):
            engine_step(fe, step)
        torch.cuda.synchronize()
        assert torch.equal(fe.flat_param, eng.flat_param), f"graph={graph}: resumed run differs from the uninterrupted one"
        for b1, b2 in zip(fe.buckets, eng.buckets):
            for t1, t2 in zip(fe._state(b1), eng._state(b2)):
                assert torch.equal(t1, t2), f"graph={graph}: resumed optimizer state differs"
        assert eng.comm.status() == 0
        print(f"rank {RANK}: engine (graph={graph}) vs torch AdamW: rel L2 of updates {total:.2e} total, {worst:.2e} worst "
              f"tensor; resume from step 3 bit-identical", flush=True)
        del eng, fe
    # a bf16 fused model trains
    from bagua_net_b200.parallel import BnetDDP

    for graph in (False, True):
        torch.manual_seed(1)
        m2 = build_model("vgg16", fused=True, **KW).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
        e2 = BnetDDP(m2, lr=1e-3, weight_decay=0.01, bucket_mb=0.25, optimizer="adamw")
        e2.enable_cuda_graph(graph)
        torch.manual_seed(5 + RANK)
        x = torch.randn(8, 3, 32, 32, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 10, (8,), device="cuda")
        ls = [float(e2.train_step(x, y)) for _ in range(25)]
        assert ls[-1] < ls[0] - 0.1 and all(v == v and abs(v) < 1e4 for v in ls), ls
        assert same_on_every_rank(e2.flat_param), "ranks hold different parameters"
        print(f"rank {RANK}: bf16 AdamW engine (graph={graph}) loss {ls[0]:.3f} -> {ls[-1]:.3f}", flush=True)
    teardown()


JOBS = {k[4:]: v for k, v in globals().items() if k.startswith("job_")}

if __name__ == "__main__":
    JOBS[sys.argv[1]]()

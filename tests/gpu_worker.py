"""Per-rank bodies of the GPU tests (launched by tests/test_gpu.py, one process per GPU)."""
from __future__ import annotations

import os
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

QUICK = os.environ.get("BNET_TEST_QUICK") == "1"      # under compute-sanitizer: same code paths, smaller tensors
RANK = int(os.environ.get("RANK", "0"))
WORLD = int(os.environ.get("WORLD_SIZE", "1"))
LOCAL = int(os.environ.get("LOCAL_RANK", "0"))


def setup(backend="nccl"):
    torch.cuda.set_device(LOCAL)
    if WORLD > 1:
        dist.init_process_group(backend)


def teardown():
    if WORLD > 1 and dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()


# ------------------------------------------------------------------ executor (transport kernels)
def job_executor():
    from bagua_net_b200.ops import P2PExecutor
    from bagua_net_b200.utils import native

    torch.cuda.set_device(0)
    ex = P2PExecutor(0)
    g = torch.Generator(device="cuda").manual_seed(1)
    # copy: sizes around vector/chunk boundaries, unaligned offsets on both sides
    for n in ([1, 15, 17, 4095, 262144 + 3] if QUICK else [1, 15, 16, 17, 4095, 65536, 262144 + 3, 1 << 20, (4 << 20) + 13, 32 << 20]):
        for so, do in [(0, 0), (1, 1), (3, 7), (16, 4)]:
            src = torch.randint(0, 256, (n + 64,), device="cuda", dtype=torch.uint8, generator=g)
            dst = torch.zeros(n + 64, device="cuda", dtype=torch.uint8)
            ex.run("copy", src[so:so + n], dst[do:do + n])
            torch.cuda.synchronize()
            assert torch.equal(dst[do:do + n], src[so:so + n]), f"copy mismatch n={n} so={so} do={do}"
            assert int(dst[:do].sum()) == 0 and int(dst[do + n:].sum()) == 0, f"copy wrote outside n={n}"
    # many jobs in flight (queue depth, round-robin over clusters)
    srcs = [torch.randn(100003 + 17 * i, device="cuda") for i in range(40)]
    dsts = [torch.empty_like(s) for s in srcs]
    torch.cuda.synchronize()
    tickets = [ex.submit("copy", s, d, sync=False) for s, d in zip(srcs, dsts)]
    for t in tickets:
        ex.wait(t)
    torch.cuda.synchronize()
    for s, d in zip(srcs, dsts):
        assert torch.equal(s, d)
    # fused accumulate / cast vs fp32 reference
    for n in [8, 1000, 4096, (1 << 20) + 8]:
        a = torch.randn(n, device="cuda")
        b = torch.randn(n, device="cuda")
        ref = a + b
        ex.run("red_add_f32", a, b)              # b += a
        torch.cuda.synchronize()
        assert torch.allclose(b, ref, rtol=0, atol=1e-6), "red_add_f32"
        h = torch.randn(n, device="cuda").to(torch.bfloat16)
        f = torch.empty(n, device="cuda")
        ex.run("cast_bf16_to_f32", h, f)
        torch.cuda.synchronize()
        assert torch.equal(f, h.float()), "cast_bf16_to_f32"
        h2 = torch.empty(n, device="cuda", dtype=torch.bfloat16)
        ex.run("cast_f32_to_bf16", a, h2)
        torch.cuda.synchronize()
        assert torch.equal(h2, a.to(torch.bfloat16)), "cast_f32_to_bf16"
        acc = torch.randn(n, device="cuda")
        ref = acc + h.float()
        ex.run("acc_bf16_to_f32", h, acc)        # acc += float(h): move + cast + accumulate in one pass
        torch.cuda.synchronize()
        assert torch.allclose(acc, ref, rtol=0, atol=1e-6), "acc_bf16_to_f32"
        x = torch.randn(n, device="cuda").to(torch.bfloat16)
        y = torch.randn(n, device="cuda").to(torch.bfloat16)
        ref = (x.float() + y.float())
        ex.run("red_add_bf16", x, y)
        torch.cuda.synchronize()
        assert torch.allclose(y.float(), ref, rtol=1e-2, atol=1e-2), "red_add_bf16"
    # fp8 (e4m3) gradient compression: quantise while moving, de-quantise + accumulate on arrival
    if hasattr(torch, "float8_e4m3fn"):
        for n in [64, 4096, (1 << 20) + 64]:
            h = (torch.randn(n, device="cuda") * 3).to(torch.bfloat16)
            scale = 16.0
            q = torch.empty(n, device="cuda", dtype=torch.uint8)
            ex.run("cast_bf16_to_e4m3", h, q, scale=scale)
            torch.cuda.synchronize()
            ref_q = (h.float() * scale).clamp(-448, 448).to(torch.float8_e4m3fn)
            assert torch.equal(q.view(torch.float8_e4m3fn).float(), ref_q.float()), "cast_bf16_to_e4m3"
            f32 = torch.randn(n, device="cuda")
            q2 = torch.empty(n, device="cuda", dtype=torch.uint8)
            ex.run("cast_f32_to_e4m3", f32, q2, scale=scale)
            torch.cuda.synchronize()
            assert torch.equal(q2.view(torch.float8_e4m3fn).float(), (f32 * scale).clamp(-448, 448).to(torch.float8_e4m3fn).float())
            acc = torch.randn(n, device="cuda")
            ref = acc + ref_q.float() / scale
            ex.run("acc_e4m3_to_f32", q, acc, scale=1.0 / scale)
            torch.cuda.synchronize()
            assert torch.allclose(acc, ref, rtol=1e-6, atol=1e-6), "acc_e4m3_to_f32"
    # bandwidth line (device-local copy through the transport kernel)
    big = torch.empty(256 << 20, device="cuda", dtype=torch.uint8).random_(0, 255)
    out = torch.empty_like(big)
    ex.run("copy", big, out)
    t0 = time.perf_counter()
    for _ in range(5):
        ex.run("copy", big, out)
    dt = (time.perf_counter() - t0) / 5
    print(f"executor env={ {k: v for k, v in os.environ.items() if k.startswith('BNET_')} } "
          f"local copy {big.numel() / dt / 1e9:.1f} GB/s (x2 traffic) stats={native.exec_stats()}", flush=True)


def job_executor_e5m2():
    """fp8 e5m2 variants of the compression ops (wide range, 2 mantissa bits) vs torch.float8_e5m2."""
    from bagua_net_b200.ops import P2PExecutor

    torch.cuda.set_device(0)
    ex = P2PExecutor(0)
    for n in [64, 4096, (1 << 20) + 64]:
        h = (torch.randn(n, device="cuda") * 3).to(torch.bfloat16)
        scale = 16.0
        q = torch.empty(n, device="cuda", dtype=torch.uint8)
        ex.run("cast_bf16_to_e5m2", h, q, scale=scale)
        torch.cuda.synchronize()
        ref_q = (h.float() * scale).clamp(-57344, 57344).to(torch.float8_e5m2)
        assert torch.equal(q.view(torch.float8_e5m2).float(), ref_q.float()), "cast_bf16_to_e5m2"
        f32 = torch.randn(n, device="cuda")
        q2 = torch.empty(n, device="cuda", dtype=torch.uint8)
        ex.run("cast_f32_to_e5m2", f32, q2, scale=scale)
        torch.cuda.synchronize()
        assert torch.equal(q2.view(torch.float8_e5m2).float(), (f32 * scale).clamp(-57344, 57344).to(torch.float8_e5m2).float())
        acc = torch.randn(n, device="cuda")
        ref = acc + ref_q.float() / scale
        ex.run("acc_e5m2_to_f32", q, acc, scale=1.0 / scale)
        torch.cuda.synchronize()
        assert torch.allclose(acc, ref, rtol=1e-6, atol=1e-6), "acc_e5m2_to_f32"
    print("e5m2 ok", flush=True)


def job_executor_decompress():
    """fp8 -> fp32 plain decompression (the all-gather half of the compressed all-reduce: overwrites instead of accumulating).
    A job of its own, run LAST by the test file: these ops were added after the round's last hardware session."""
    from bagua_net_b200.ops import P2PExecutor

    torch.cuda.set_device(0)
    ex = P2PExecutor(0)
    for name, fp8, lim in (("e4m3", torch.float8_e4m3fn, 448.0), ("e5m2", torch.float8_e5m2, 57344.0)):
        for n in [64, 4096, (1 << 20) + 64, 777]:
            h = (torch.randn(n, device="cuda") * 3).to(torch.bfloat16)
            scale = 16.0
            ref_q = (h.float() * scale).clamp(-lim, lim).to(fp8)
            q = ref_q.view(torch.uint8).clone()
            dec = torch.full((n,), 7.0, device="cuda")
            ex.run(f"cast_{name}_to_f32", q, dec, scale=1.0 / scale)
            torch.cuda.synchronize()
            assert torch.equal(dec, ref_q.float() / scale), f"cast_{name}_to_f32 n={n}"
    print("fp8 decompression ok", flush=True)


def job_executor_idle():
    from bagua_net_b200.ops import P2PExecutor
    from bagua_net_b200.utils import native

    torch.cuda.set_device(0)
    ex = P2PExecutor(0)
    a = torch.randn(1 << 16, device="cuda")
    b = torch.empty_like(a)
    for i in range(6):
        b.zero_()
        ex.run("copy", a, b)
        torch.cuda.synchronize()                 # returns only after the parked kernel has left
        assert torch.equal(a, b)
        time.sleep(0.01)                         # > idle timeout: next job needs a relaunch
    st = native.exec_stats()
    assert st["launches"] >= 3, st
    print("idle/relaunch ok", st, flush=True)


# ------------------------------------------------------------------ fused SGD
def _sgd_reference(p32, g_list, lr, mu, wd, steps):
    buf = torch.zeros_like(p32)
    p = p32.clone()
    for s in range(steps):
        g = torch.stack([x.float() for x in g_list[s]]).sum(0) / len(g_list[s])
        dp = g + wd * p
        buf = mu * buf + dp
        p = p - lr * buf
    return p


def job_fused_sgd():
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(256 << 20)
    for dtype in (torch.bfloat16, torch.float32):
        n = 8 * WORLD * 4099
        torch.manual_seed(7)
        p0 = (torch.randn(n, device="cuda") * 0.1)
        param = comm.alloc(n, dtype)
        grad = comm.alloc(n, dtype)
        param.copy_(p0.to(dtype))
        shard = n // WORLD
        master = param[RANK * shard:(RANK + 1) * shard].float().contiguous()
        mom = torch.zeros_like(master)
        lr, mu, wd, steps = 0.1, 0.9, 0.01, 4
        all_g = []
        for s in range(steps):
            gs = []
            for r in range(WORLD):
                torch.manual_seed(100 * s + r)
                gs.append((torch.randn(n, device="cuda")).to(dtype))
            all_g.append(gs)
        for s in range(steps):
            grad.copy_(all_g[s][RANK])
            torch.cuda.synchronize()
            if WORLD > 1:
                dist.barrier()
            comm.fused_allreduce_sgd(grad, param, master, mom, lr, mu, wd, zero_grads=True)
            torch.cuda.synchronize()
            assert int((grad != 0).sum()) == 0, "gradients were not re-zeroed"
        ref = _sgd_reference(p0.to(dtype).float(), all_g, lr, mu, wd, steps)
        # fp32 master stays close to the fp32 reference (bf16 only rounds the reduced gradient)
        err_m = (master - ref[RANK * shard:(RANK + 1) * shard]).abs().max().item()
        tol = 3e-2 if dtype == torch.bfloat16 else 1e-5
        assert err_m < tol, f"{dtype} master err {err_m}"
        err_p = (param.float() - ref).abs().max().item()
        assert err_p < (6e-2 if dtype == torch.bfloat16 else 1e-5), f"{dtype} param err {err_p}"
        if WORLD > 1:   # every rank holds identical parameters
            chk = param.float().sum().double().reshape(1)
            lst = [torch.zeros_like(chk) for _ in range(WORLD)]
            dist.all_gather(lst, chk)
            assert all(torch.equal(lst[0], x) for x in lst), "ranks diverged"
        print(f"rank {RANK}: fused sgd {dtype} ok (master err {err_m:.2e}, param err {err_p:.2e}, "
              f"multicast={comm.has_multicast})", flush=True)
    assert comm.status() == 0
    teardown()


# ------------------------------------------------------------------ DDP engine vs torch DDP semantics
def job_ddp_engine():
    from bagua_net_b200.models import build_model
    from bagua_net_b200.parallel import BnetDDP

    setup()
    torch.backends.cudnn.allow_tf32 = False          # compare against torch SGD at full fp32 precision
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    kw = dict(width_div=8, fc_dim=128, image_size=32, num_classes=10, dropout=0.0)
    model = build_model("vgg16", **kw).cuda()
    ref = build_model("vgg16", **kw).cuda()
    ref.load_state_dict(model.state_dict())
    model = model.to(memory_format=torch.channels_last)
    lr, mu, wd = 0.05, 0.9, 1e-4
    eng = BnetDDP(model, lr=lr, momentum=mu, weight_decay=wd, bucket_mb=0.25)
    assert len(eng.buckets) > 1
    opt = torch.optim.SGD(ref.parameters(), lr=lr, momentum=mu, weight_decay=wd)
    losses, ref_losses = [], []
    for step in range(6):
        xs, ys = [], []
        for r in range(WORLD):
            torch.manual_seed(1000 + 10 * step + r)
            xs.append(torch.randn(4, 3, 32, 32, device="cuda"))
            ys.append(torch.randint(0, 10, (4,), device="cuda"))
        losses.append(float(eng.train_step(xs[RANK].contiguous(memory_format=torch.channels_last), ys[RANK])))
        # reference: full global batch on one model == averaged per-rank gradients
        opt.zero_grad()
        loss = torch.nn.functional.cross_entropy(ref(torch.cat(xs)), torch.cat(ys))
        loss.backward()
        opt.step()
        ref_losses.append(float(torch.nn.functional.cross_entropy(ref(xs[RANK]), ys[RANK]).item()))
    torch.cuda.synchronize()
    worst = 0.0
    for (n1, p1), (n2, p2) in zip(model.named_parameters(), ref.named_parameters()):
        worst = max(worst, (p1.float() - p2.float()).abs().max().item())
    assert worst < 1e-3, f"fp32 engine diverged from torch SGD: {worst}"
    assert eng.kernel_launches >= 6 * len(eng.buckets)
    print(f"rank {RANK}: ddp engine fp32 matches torch SGD (max param diff {worst:.2e}); losses {losses[:3]}...", flush=True)
    # bf16 variant trains (loss goes down on a fixed batch)
    torch.manual_seed(1)
    m2 = build_model("vgg16", **kw).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    e2 = BnetDDP(m2, lr=0.02, momentum=0.9, weight_decay=0.0, bucket_mb=0.25)
    torch.manual_seed(5 + RANK)
    x = torch.randn(8, 3, 32, 32, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (8,), device="cuda")
    ls = [float(e2.train_step(x, y)) for _ in range(25)]
    assert ls[-1] < ls[0] - 0.1 and all(x == x for x in ls), ls
    xh, yh = x.cpu().pin_memory(), y.cpu().pin_memory()
    assert isinstance(e2.train_step_from_host(xh, yh), float)
    print(f"rank {RANK}: bf16 engine loss {ls[0]:.3f} -> {ls[-1]:.3f}", flush=True)
    # CUDA-graph mode: the whole step (both streams, the cross-rank kernels included) replays as one graph
    torch.manual_seed(1)
    m3 = build_model("vgg16", fused=True, **kw).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    e3 = BnetDDP(m3, lr=0.02, momentum=0.9, weight_decay=0.0, bucket_mb=0.25)
    e3.enable_cuda_graph(True)
    before = e3.kernel_launches
    lg = [float(e3.train_step(x, y)) for _ in range(25)]
    assert lg[-1] < lg[0] - 0.1 and all(v == v for v in lg), lg
    assert e3._graph is not None and e3.kernel_launches - before >= 25 * len(e3.buckets)
    assert isinstance(e3.train_step_from_host(xh, yh), float)
    print(f"rank {RANK}: graph engine loss {lg[0]:.3f} -> {lg[-1]:.3f}", flush=True)
    assert eng.comm.status() == 0 and e2.comm.status() == 0 and e3.comm.status() == 0
    teardown()


def job_ddp_api():
    """Loader-facing loop (prefetched H2D copies) and checkpoint / resume of the engine, eager and graph mode."""
    from bagua_net_b200.models import build_model
    from bagua_net_b200.parallel import BnetDDP

    setup()
    kw = dict(width_div=8, fc_dim=128, image_size=32, num_classes=10, dropout=0.0)
    for graph in (False, True):
        torch.manual_seed(1)
        m3 = build_model("vgg16", fused=True, **kw).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
        e3 = BnetDDP(m3, lr=0.02, momentum=0.9, weight_decay=0.0, bucket_mb=0.25)
        e3.enable_cuda_graph(graph)
        torch.manual_seed(5 + RANK)
        x = torch.randn(8, 3, 32, 32, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
        y = torch.randint(0, 10, (8,), device="cuda")
        xh, yh = x.cpu().pin_memory(), y.cpu().pin_memory()
        lg = [float(e3.train_step(x, y)) for _ in range(10)]
        # loader-facing loop with the next batch's H2D copy prefetched: one loss per batch, training continues
        lp = list(e3.train_from_host((xh, yh) for _ in range(6)))
        assert len(lp) == 6 and all(isinstance(v, float) and v == v for v in lp) and max(lp) < lg[0] + 1.0, lp
        assert list(e3.train_from_host(iter(()))) == []
        # checkpoint / resume: weights through the module, optimizer shards through the engine
        weights = {k: v.clone() for k, v in m3.state_dict().items()}
        opt = e3.optimizer_state_dict()
        after = float(e3.train_step(x, y))
        m3.load_state_dict(weights)
        e3.load_optimizer_state_dict(opt)
        torch.cuda.synchronize()
        again = float(e3.train_step(x, y))
        assert abs(again - after) < 5e-2, (after, again)    # same state, same batch -> same loss (bf16 tolerance)
        assert e3.comm.status() == 0
        print(f"rank {RANK}: ddp api ok (graph={graph}) losses {lp[:2]}... resume {after:.4f} vs {again:.4f}", flush=True)
    teardown()


def job_lr_schedule():
    """set_lr: hyper-parameters move to device memory; eager engine == torch SGD under a per-step schedule, and a captured
    graph follows the schedule without being re-captured."""
    from bagua_net_b200.models import build_model
    from bagua_net_b200.parallel import BnetDDP

    setup()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    kw = dict(width_div=8, fc_dim=128, image_size=32, num_classes=10, dropout=0.0)
    model = build_model("vgg16", **kw).cuda()
    ref = build_model("vgg16", **kw).cuda()
    ref.load_state_dict(model.state_dict())
    model = model.to(memory_format=torch.channels_last)
    mu, wd = 0.9, 1e-4
    eng = BnetDDP(model, lr=0.05, momentum=mu, weight_decay=wd, bucket_mb=0.25)
    opt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=mu, weight_decay=wd)
    for step in range(5):
        lr = 0.05 * (0.7 ** step)
        eng.set_lr(lr)
        for g in opt.param_groups:
            g["lr"] = lr
        xs, ys = [], []
        for r in range(WORLD):
            torch.manual_seed(2000 + 10 * step + r)
            xs.append(torch.randn(4, 3, 32, 32, device="cuda"))
            ys.append(torch.randint(0, 10, (4,), device="cuda"))
        eng.train_step(xs[RANK].contiguous(memory_format=torch.channels_last), ys[RANK])
        opt.zero_grad()
        torch.nn.functional.cross_entropy(ref(torch.cat(xs)), torch.cat(ys)).backward()
        opt.step()
    torch.cuda.synchronize()
    worst = max((p1.float() - p2.float()).abs().max().item() for p1, p2 in zip(model.parameters(), ref.parameters()))
    assert worst < 1e-3, f"engine with a learning-rate schedule diverged from torch SGD: {worst}"
    # graph mode: one re-capture when the schedule starts, none afterwards
    torch.manual_seed(1)
    m2 = build_model("vgg16", fused=True, **kw).cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    e2 = BnetDDP(m2, lr=0.02, momentum=0.9, weight_decay=0.0, bucket_mb=0.25)
    e2.enable_cuda_graph(True)
    x = torch.randn(8, 3, 32, 32, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (8,), device="cuda")
    l0 = float(e2.train_step(x, y))
    e2.set_lr(0.02)
    float(e2.train_step(x, y))
    g = e2._graph
    for step in range(20):
        e2.set_lr(0.02 * (0.97 ** step))
        last = float(e2.train_step(x, y))
        assert e2._graph is g, "the graph was re-captured for a learning-rate change"
    assert last == last and last < l0, (l0, last)
    e2.set_lr(0.0)                       # lr = 0: parameters must stop moving
    before = e2.flat_param.clone()
    float(e2.train_step(x, y))
    torch.cuda.synchronize()
    assert torch.equal(before, e2.flat_param), "lr=0 in device memory was not honoured by the captured step"
    print(f"rank {RANK}: lr schedule ok (max diff {worst:.2e})", flush=True)
    teardown()


def job_collectives_any():
    """all_reduce / broadcast / all_gather / reduce_scatter on ordinary (non-heap) tensors vs torch.distributed."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(4 << 20)               # small heap: the 4-6 MB tensors below need several staging chunks
    torch.manual_seed(100 + RANK)
    for dtype, n in ((torch.float32, 1), (torch.float32, 1000003), (torch.bfloat16, 4099), (torch.bfloat16, 3 << 20)):
        x = torch.randn(n, device="cuda").to(dtype)
        ref = x.float().clone()
        if WORLD > 1:
            dist.all_reduce(ref)
        got = comm.all_reduce_tensor(x.clone())
        tol = 1e-5 if dtype == torch.float32 else 3e-2
        assert torch.allclose(got.float(), ref, rtol=tol, atol=tol), f"all_reduce_tensor {dtype} n={n}"
        b = x.clone()
        comm.broadcast_tensor(b, src=WORLD - 1)
        refb = x.clone()
        if WORLD > 1:
            dist.broadcast(refb, src=WORLD - 1)
        assert torch.equal(b, refb), f"broadcast_tensor {dtype} n={n}"
        ag = comm.all_gather_tensor(x)
        refs = [torch.empty_like(x) for _ in range(WORLD)]
        if WORLD > 1:
            dist.all_gather(refs, x)
        else:
            refs = [x]
        assert torch.equal(ag, torch.stack(refs)), f"all_gather_tensor {dtype} n={n}"
    y = torch.randn(WORLD * 50001, device="cuda")
    rs = comm.reduce_scatter_tensor(y)
    ref = y.clone()
    if WORLD > 1:
        dist.all_reduce(ref)
    assert torch.allclose(rs, ref.view(WORLD, -1)[RANK], rtol=1e-5, atol=1e-5), "reduce_scatter_tensor"
    m = torch.randn(5, 7, device="cuda").t()          # non-contiguous input
    refm = m.contiguous()                              # (torch's own all_reduce wants a contiguous tensor)
    if WORLD > 1:
        dist.all_reduce(refm)
    assert torch.allclose(comm.all_reduce_tensor(m.clone()), refm, rtol=1e-5, atol=1e-5)
    torch.cuda.synchronize()
    assert comm.status() == 0
    print(f"rank {RANK}: collectives on ordinary tensors ok", flush=True)
    teardown()


def job_fused_nn():
    """ConvBiasReLU / ConvBiasReLUPool vs the eager PyTorch chain, forward and backward."""
    from bagua_net_b200.ops import fused_nn
    from bagua_net_b200.ops.fused_nn import ConvBiasReLU

    torch.cuda.set_device(0)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    for dtype, tol in ((torch.float32, 2e-4), (torch.bfloat16, 6e-2)):
        for (cin, cout, hw, pool) in [(3, 64, 32, False), (64, 64, 32, True), (16, 128, 20, True), (32, 512, 14, False),
                                      (8, 24 if dtype == torch.float32 else 40, 10, True)]:
            torch.manual_seed(cin * 7 + cout)
            blk = ConvBiasReLU(cin, cout, 3, 1, 1, pool=pool).cuda().to(dtype).to(memory_format=torch.channels_last)
            ref = torch.nn.Conv2d(cin, cout, 3, 1, 1).cuda().float()
            ref.weight.data.copy_(blk.conv.weight.data.float())
            ref.bias.data.copy_(blk.conv.bias.data.float())
            x = torch.randn(4, cin, hw, hw, device="cuda")
            xa = x.to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(cin != 3)
            xb = xa.detach().float().requires_grad_(cin != 3)
            before = fused_nn.LAUNCHES
            ya = blk(xa)
            yb = torch.relu(ref(xb))
            if pool:
                yb = torch.nn.functional.max_pool2d(yb, 2, 2)
            assert fused_nn.LAUNCHES > before, "fused kernel did not run"
            assert ya.shape == yb.shape
            err = (ya.float() - yb).abs().max().item()
            assert err < tol * max(1.0, yb.abs().max().item()), f"fwd {dtype} {cin}->{cout} pool={pool}: {err}"
            g = torch.randn_like(yb)
            ya.backward(g.to(dtype))
            yb.backward(g.to(dtype).float())
            torch.cuda.synchronize()
            for name, a_, b_ in (("w", blk.conv.weight.grad, ref.weight.grad), ("b", blk.conv.bias.grad, ref.bias.grad)) + (
                    (("x", xa.grad, xb.grad),) if cin != 3 else ()):
                e = (a_.float() - b_).abs().max().item()
                scale = max(1.0, b_.abs().max().item())
                if dtype == torch.float32:
                    assert e < tol * scale, f"bwd {name} {dtype} {cin}->{cout} pool={pool}: {e} / {scale}"
                else:
                    # bf16: ReLU masks / pool arg-max come from bf16-rounded activations, so a few
                    # near-ties route their gradient differently than the fp32 reference: compare in L2
                    rel = ((a_.float() - b_).norm() / b_.norm().clamp_min(1e-6)).item()
                    assert rel < 0.06, f"bwd {name} {dtype} {cin}->{cout} pool={pool}: rel L2 {rel}"
    # whole model: fused VGG == eager VGG in fp32
    from bagua_net_b200.models import build_model

    kw = dict(width_div=8, fc_dim=64, image_size=32, num_classes=10, dropout=0.0)
    torch.manual_seed(3)
    a = build_model("vgg16", fused=True, **kw).cuda().to(memory_format=torch.channels_last)
    b = build_model("vgg16", fused=False, **kw).cuda()
    for pa, pb in zip(a.parameters(), b.parameters()):
        pb.data.copy_(pa.data)
    x = torch.randn(4, 3, 32, 32, device="cuda")
    y = torch.randint(0, 10, (4,), device="cuda")
    la = torch.nn.functional.cross_entropy(a(x.contiguous(memory_format=torch.channels_last)), y)
    lb = torch.nn.functional.cross_entropy(b(x), y)
    la.backward()
    lb.backward()
    assert abs(la.item() - lb.item()) < 1e-4, (la.item(), lb.item())
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert (pa.grad - pb.grad).abs().max().item() < 1e-3 * max(1.0, pb.grad.abs().max().item())
    assert fused_nn.self_check(verbose=True), "the self-check bench.py relies on disagrees with the detailed comparison above"
    print("fused_nn ok", flush=True)


def job_fused_bn():
    """conv_bn_act (training-mode BatchNorm + ReLU + residual fused behind a convolution) vs the eager chain."""
    import copy

    from bagua_net_b200.models import build_model
    from bagua_net_b200.ops import fused_nn
    from bagua_net_b200.ops.fused_nn import conv_bn_act

    torch.cuda.set_device(0)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    for dtype, tol in ((torch.float32, 2e-3), (torch.bfloat16, 6e-2)):
        for (cin, cout, hw, k, stride, relu, with_res) in [(3, 64, 32, 7, 2, True, False), (64, 64, 16, 3, 1, True, False),
                                                          (64, 256, 16, 1, 1, True, True), (256, 512, 8, 1, 2, False, False),
                                                          (128, 2048, 4, 1, 1, True, True)]:
            if dtype == torch.float32 and cout > 1024:
                continue                      # fp32: 4 channels per vector, at most 1024 channels
            torch.manual_seed(cin + cout)
            conv = torch.nn.Conv2d(cin, cout, k, stride, k // 2, bias=False).cuda().to(dtype).to(memory_format=torch.channels_last)
            bn_a = torch.nn.BatchNorm2d(cout).cuda().to(dtype)
            with torch.no_grad():
                bn_a.weight.copy_(torch.rand(cout) + 0.5)
                bn_a.bias.copy_(torch.randn(cout) * 0.1)
            bn_b = copy.deepcopy(bn_a)
            x = torch.randn(6, cin, hw, hw, device="cuda").to(dtype).contiguous(memory_format=torch.channels_last)
            ho = (hw + 2 * (k // 2) - k) // stride + 1
            res = torch.randn(6, cout, ho, ho, device="cuda").to(dtype).contiguous(memory_format=torch.channels_last) if with_res else None
            xa, xb = x.clone().requires_grad_(cin != 3), x.clone().requires_grad_(cin != 3)
            ra = res.clone().requires_grad_(True) if with_res else None
            rb = res.clone().requires_grad_(True) if with_res else None
            before = fused_nn.LAUNCHES
            ya = conv_bn_act(xa, conv, bn_a, relu=relu, res=ra)
            assert fused_nn.LAUNCHES == before + 2, "fused BatchNorm kernels did not run"
            go = torch.randn_like(ya)
            ya.backward(go)
            ga = {"w": conv.weight.grad.float().clone(), "gamma": bn_a.weight.grad.float().clone(), "beta": bn_a.bias.grad.float().clone()}
            if cin != 3:
                ga["x"] = xa.grad.float().clone()
            if with_res:
                ga["res"] = ra.grad.float().clone()
            conv.zero_grad(set_to_none=True)
            yb = bn_b(conv(xb))
            if with_res:
                yb = yb + rb
            if relu:
                yb = torch.relu(yb)
            yb.backward(go)
            gb = {"w": conv.weight.grad.float(), "gamma": bn_b.weight.grad.float(), "beta": bn_b.bias.grad.float()}
            if cin != 3:
                gb["x"] = xb.grad.float()
            if with_res:
                gb["res"] = rb.grad.float()
            torch.cuda.synchronize()
            rel = lambda a, b: ((a - b).norm() / b.norm().clamp_min(1e-6)).item()      # noqa: E731
            e = rel(ya.float(), yb.float())
            assert e < tol, f"fwd {dtype} {cin}->{cout}: {e}"
            for name in ga:
                e = rel(ga[name], gb[name])
                assert e < tol, f"bwd {name} {dtype} {cin}->{cout} k{k} relu={relu} res={with_res}: {e}"
            assert rel(bn_a.running_mean.float(), bn_b.running_mean.float()) < tol
            assert rel(bn_a.running_var.float(), bn_b.running_var.float()) < tol
            assert int(bn_a.num_batches_tracked) == int(bn_b.num_batches_tracked) == 1
    assert fused_nn.self_check_bn(verbose=True)
    # whole model: fused ResNet-18 == eager ResNet-18 in fp32 (same weights, same batch)
    torch.manual_seed(5)
    a = build_model("resnet18", fused=True, num_classes=10).cuda().to(memory_format=torch.channels_last)
    b = build_model("resnet18", num_classes=10).cuda()
    b.load_state_dict(a.state_dict())
    x = torch.randn(8, 3, 64, 64, device="cuda")
    y = torch.randint(0, 10, (8,), device="cuda")
    la = torch.nn.functional.cross_entropy(a(x.contiguous(memory_format=torch.channels_last)), y)
    lb = torch.nn.functional.cross_entropy(b(x), y)
    la.backward()
    lb.backward()
    assert abs(la.item() - lb.item()) < 1e-3, (la.item(), lb.item())
    for (n1, pa), (n2, pb) in zip(a.named_parameters(), b.named_parameters()):
        e = ((pa.grad - pb.grad).norm() / pb.grad.norm().clamp_min(1e-6)).item()
        assert e < 2e-2, f"resnet18 grad {n1}: {e}"
    print("fused_bn ok", flush=True)


def job_tc_linear():
    """wgmma linear (csrc/cuda/tc_gemm.cu) vs an fp32 PyTorch reference: both operand orientations, ragged M/N/K,
    bias, ReLU, non-trivial row pitches, and the autograd wrapper."""
    from bagua_net_b200.ops import tc_linear

    setup()
    assert tc_linear.supported(), "wgmma linear reports unsupported on this GPU / driver"
    assert tc_linear.self_check(verbose=True), "tc_linear self-check failed"
    torch.manual_seed(3)
    for (M, N, K) in [(1, 8, 8), (32, 4096, 25088), (64, 1000, 4096), (65, 520, 200), (512, 512, 4096), (1000, 1000, 1000)]:
        x = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        for relu, splits in ((False, 1), (True, 1), (True, None), (False, 3)):   # fused epilogue; automatic / forced split-K
            y = tc_linear.linear(x, w, b, relu, splits=splits)
            assert tc_linear.last_error() == 0, f"watchdog tripped at {M}x{N}x{K}"
            ref = x.float() @ w.float().t() + b.float()
            ref = torch.relu(ref) if relu else ref
            err = (y.float() - ref).abs().max().item()
            assert err < 0.08, f"tc_linear {M}x{N}x{K} relu={relu} splits={splits}: max abs err {err}"
    # the backward GEMMs: W, gY and X read MN-major, both orientations of dX, ragged extents
    for (M, N, K) in [(32, 4096, 1024), (64, 136, 264), (200, 72, 520), (512, 1024, 768), (1000, 1000, 1000)]:
        gy = torch.randn(M, N, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") / N ** 0.5).bfloat16()
        x = torch.randn(M, K, device="cuda").bfloat16()
        dx, dw = tc_linear.linear_dgrad(gy, w), tc_linear.linear_wgrad(gy, x)
        assert tc_linear.last_error() == 0, f"watchdog tripped in the backward GEMMs at {M}x{N}x{K}"
        e1 = (dx.float() - gy.float() @ w.float()).abs().max().item()
        ref = gy.float().t() @ x.float()
        e2 = ((dw.float() - ref).abs().max() / ref.abs().max()).item()
        assert e1 < 0.1 and e2 < 0.02, f"backward {M}x{N}x{K}: dgrad abs err {e1}, wgrad rel err {e2}"
    # strided views (row pitch != K), no bias
    big = torch.randn(96, 1024, device="cuda").bfloat16()
    x, w = big[:40, 128:640], big[40:, 128:640]
    y = tc_linear.linear(x, w)
    assert tc_linear.last_error() == 0
    assert (y.float() - x.float() @ w.float().t()).abs().max().item() < 0.5
    # autograd wrapper against eager
    x = torch.randn(32, 256, device="cuda").bfloat16().requires_grad_()
    w = (torch.randn(128, 256, device="cuda") / 16).bfloat16().requires_grad_()
    b = torch.randn(128, device="cuda").bfloat16().requires_grad_()
    y = tc_linear.linear_bias_act(x, w, b, True)
    y.float().square().sum().backward()
    x2, w2, b2 = (t.detach().clone().requires_grad_() for t in (x, w, b))
    torch.relu(torch.nn.functional.linear(x2, w2, b2)).float().square().sum().backward()
    for a, r, name in ((x.grad, x2.grad, "dx"), (w.grad, w2.grad, "dw"), (b.grad, b2.grad, "db")):
        rel = (a.float() - r.float()).norm() / (r.float().norm() + 1e-6)
        assert rel < 0.05, f"{name}: rel err {rel}"
    print(f"tc_linear ok, launches={tc_linear.LAUNCHES}")


def job_tc_row_parallel():
    """GEMM + all-reduce in one kernel: every rank multiplies its K-shard, the epilogue adds into every rank's output."""
    from bagua_net_b200.ops import tc_linear
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(64 << 20)
    torch.manual_seed(11)                                  # same full problem on every rank
    for (M, N, K, splits) in [(32, 512, 1024, 1), (32, 512, 4096, 4), (256, 384, 2048, 1), (130, 200, 512, 2)]:
        xf = torch.randn(M, K * WORLD, device="cuda").bfloat16()
        wf = (torch.randn(N, K * WORLD, device="cuda") / (K * WORLD) ** 0.5).bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        x, w = xf[:, RANK * K:(RANK + 1) * K], wf[:, RANK * K:(RANK + 1) * K]
        out = tc_linear.row_parallel_linear(x, w, comm, bias=b, splits=splits)
        assert tc_linear.last_error() == 0, f"watchdog tripped at {M}x{N}x{K}"
        ref = xf.float() @ wf.float().t() + b.float()
        err = (out - ref).abs().max().item()
        assert err < 0.05, f"row_parallel {M}x{N}x{K} splits={splits}: max abs err {err}"
    # GEMM -> reduce-scatter: each rank keeps only its row block of the sum
    for (M, N, K, splits) in [(32 * WORLD, 512, 1024, 1), (128 * WORLD, 384, 2048, 2)]:
        xf = torch.randn(M, K * WORLD, device="cuda").bfloat16()
        wf = (torch.randn(N, K * WORLD, device="cuda") / (K * WORLD) ** 0.5).bfloat16()
        x, w = xf[:, RANK * K:(RANK + 1) * K], wf[:, RANK * K:(RANK + 1) * K]
        out = tc_linear.linear_reduce_scatter(x, w, comm, splits=splits)
        assert tc_linear.last_error() == 0
        ref = (xf.float() @ wf.float().t())[RANK * (M // WORLD):(RANK + 1) * (M // WORLD)]
        err = (out - ref).abs().max().item()
        assert err < 0.05, f"reduce_scatter {M}x{N}x{K}: max abs err {err}"
    # all-gather -> GEMM: the activation is sharded by rows, peers' shards are read by TMA over NVLink
    for (rows, N, K) in [(128, 512, 1024), (256, 1000, 520)]:
        torch.manual_seed(21)
        xf = torch.randn(rows * WORLD, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        shard = comm.alloc(rows * K, torch.bfloat16).view(rows, K)
        shard.copy_(xf[RANK * rows:(RANK + 1) * rows])
        y = tc_linear.allgather_linear(shard, w, comm, bias=b, relu=True)
        assert tc_linear.last_error() == 0
        ref = torch.relu(xf.float() @ w.float().t() + b.float())
        err = (y.float() - ref).abs().max().item()
        assert err < 0.08, f"allgather_linear {rows}x{N}x{K}: max abs err {err}"
    torch.cuda.synchronize()
    assert comm.status() == 0
    print(f"tc_row_parallel ok (multicast={comm.has_multicast})")


def job_pack_cast():
    from bagua_net_b200.ops import pack_cast
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(64 << 20)
    ts = [torch.randn(n, device="cuda") for n in (1, 7, 1024, 100003, 1 << 20)]
    total = sum(t.numel() for t in ts)
    dst = comm.alloc(total, torch.bfloat16)
    pack_cast(comm, ts, dst, scale=0.5)
    torch.cuda.synchronize()
    ref = torch.cat([(t * 0.5).to(torch.bfloat16) for t in ts])
    assert torch.equal(dst, ref)
    print("pack_cast ok", flush=True)
    teardown()


# ------------------------------------------------------------------ multi-GPU all-reduce
def job_allreduce():
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(1 << 30)
    algos = ["p2p"] + (["nvls"] if comm.has_multicast else [])
    print(f"rank {RANK}: multicast={comm.has_multicast}", flush=True)
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        for n in ([16 * WORLD, 4096 * WORLD + 16 * WORLD * 3] if QUICK else [16 * WORLD, 4096 * WORLD, (1 << 20) + 16 * WORLD * 3, 16 << 20]):
            n = n // (16 * WORLD) * (16 * WORLD)
            t = comm.alloc(n, dtype)
            torch.manual_seed(RANK + 17)
            mine = torch.randn(n, device="cuda").to(dtype)
            alls = []
            for r in range(WORLD):
                torch.manual_seed(r + 17)
                alls.append(torch.randn(n, device="cuda").to(dtype).float())
            for op in ("sum", "avg", "max", "min"):
                ref = {"sum": sum(alls), "avg": sum(alls) / WORLD, "max": torch.stack(alls).max(0).values,
                       "min": torch.stack(alls).min(0).values}[op]
                for algo in algos:
                    t.copy_(mine)
                    torch.cuda.synchronize()
                    dist.barrier()
                    comm.all_reduce(t, op, algo=algo)
                    torch.cuda.synchronize()
                    tol = 1e-5 if dtype == torch.float32 else (2e-2 if dtype == torch.bfloat16 else 4e-3)
                    err = (t.float() - ref).abs().max().item()
                    assert err <= tol * max(1.0, ref.abs().max().item()), f"{algo} {op} {dtype} n={n} err={err}"
                # one-shot, out of place
                t.copy_(mine)
                torch.cuda.synchronize()
                dist.barrier()
                out = torch.empty_like(t)
                comm.all_reduce_oneshot(t, out, op)
                torch.cuda.synchronize()
                err = (out.float() - ref).abs().max().item()
                assert err <= (1e-5 if dtype == torch.float32 else 2e-2) * max(1.0, ref.abs().max().item()), f"oneshot {op} {dtype}"
    # barrier-free small-message path: ordinary (non-heap) tensors, odd lengths, in place and out of place, many calls back to
    # back (the call counter lives on the device), and under a CUDA graph
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        for n in (1, 7, 256, 4097, 8192):
            for op in ("sum", "avg", "max", "min"):
                alls = [(((torch.arange(n, device="cuda") * 3 + r) % 11) - 5).to(dtype).float() for r in range(WORLD)]
                ref = {"sum": sum(alls), "avg": sum(alls) / WORLD, "max": torch.stack(alls).max(0).values,
                       "min": torch.stack(alls).min(0).values}[op]
                mine = alls[RANK].to(dtype)
                for rep in range(3):
                    x = mine.clone()
                    out = comm.all_reduce_ll(x, None if rep % 2 else torch.empty_like(x), op=op)
                    err = (out.float() - ref).abs().max().item()
                    assert err <= (0 if op != "avg" else 2e-2), f"ll {op} {dtype} n={n} rep={rep} err={err}"
    x = torch.full((1000,), float(RANK + 1), device="cuda", dtype=torch.float32)
    y = torch.empty_like(x)
    torch.cuda.synchronize()
    dist.barrier()
    g = torch.cuda.CUDAGraph()
    s_ = torch.cuda.Stream()
    s_.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s_):
        comm.all_reduce_ll(x, y)
    torch.cuda.current_stream().wait_stream(s_)
    with torch.cuda.graph(g):
        comm.all_reduce_ll(x, y)
    for _ in range(5):
        g.replay()
    torch.cuda.synchronize()
    assert bool((y == WORLD * (WORLD + 1) / 2).all()), "LL all-reduce under graph replay is wrong"
    x = torch.ones(512, device="cuda", dtype=torch.bfloat16)       # 1 KiB: the latency line
    for _ in range(20):
        comm.all_reduce_ll(x.clone())
    torch.cuda.synchronize()
    dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    xs = [x.clone() for _ in range(200)]
    e0.record()
    for xi in xs:
        comm.all_reduce_ll(xi)
    e1.record()
    torch.cuda.synchronize()
    if RANK == 0:
        print(f"allreduce ll 1 KiB: {e0.elapsed_time(e1) / 200 * 1e3:.2f} us per call (200 back-to-back launches, world {WORLD})", flush=True)
    # quick bandwidth lines
    for algo in ([] if QUICK else algos):
        for nbytes in (1 << 20, 64 << 20, 512 << 20):
            t = comm.alloc(nbytes // 2, torch.bfloat16)
            t.fill_(1)
            for _ in range(3):
                comm.all_reduce(t, "sum", algo=algo)
            torch.cuda.synchronize()
            dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(10):
                comm.all_reduce(t, "sum", algo=algo)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 10
            if RANK == 0:
                alg = nbytes / ms / 1e6
                print(f"allreduce {algo} {nbytes >> 20} MiB: {ms * 1e3:.1f} us algbw {alg:.1f} GB/s busbw "
                      f"{alg * 2 * (WORLD - 1) / WORLD:.1f} GB/s", flush=True)
            comm._bump -= 0   # keep allocations: heap is 1 GiB
    assert comm.status() == 0
    teardown()


def job_nccl_allreduce():
    """Stock torch.distributed all_reduce with NCCL forced through our plugin (env set by the test)."""
    setup("nccl")
    for n in (1, 1024, 1 << 20, (8 << 20) + 5):
        t = torch.full((n,), float(RANK + 1), device="cuda")
        dist.all_reduce(t)
        torch.cuda.synchronize()
        exp = float(sum(range(1, WORLD + 1)))
        assert torch.all(t == exp), f"nccl allreduce over plugin wrong for n={n}: {t[:4]}"
    b = torch.full((1 << 22,), float(RANK), device="cuda", dtype=torch.bfloat16)
    dist.all_reduce(b)
    torch.cuda.synchronize()
    assert torch.all(b.float() == float(sum(range(WORLD))))
    x = torch.randn(64 << 20, device="cuda")
    for _ in range(3):
        dist.all_reduce(x)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(5):
        dist.all_reduce(x)
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / 5
    if RANK == 0:
        from bagua_net_b200.utils import native

        print(f"nccl-over-plugin allreduce 256 MiB: algbw {x.numel() * 4 / dt / 1e9:.2f} GB/s exec={native.exec_stats()}",
              flush=True)
    teardown()


def job_fused_sgd_staggered():
    """The race the advisor found (round 1): with many CTAs per rank and a compute kernel hogging the SMs, CTAs of the
    fused all-reduce + SGD kernel start staggered, and a CTA that zeroes gradients another CTA's pairing reads would
    corrupt the reduction.  nb = 64 blocks on a bucket whose per-rank share is not a multiple of the grid stride."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    comm = SymmComm(512 << 20)
    n = 8 * WORLD * (64 * 512 * 5 + 4099)          # per-rank vectors: NOT a multiple of 64 blocks x 512 threads
    dtype = torch.bfloat16
    param, grad = comm.alloc(n, dtype), comm.alloc(n, dtype)
    shard = n // WORLD
    master = torch.zeros(shard, device="cuda", dtype=torch.float32)
    mom = torch.zeros_like(master)
    side = torch.cuda.Stream()
    a = torch.randn(8192, 8192, device="cuda", dtype=torch.bfloat16)
    for step in range(6):
        # small integers: the sum over ranks is exact in bf16, so ANY lost or doubled contribution shows
        grad.copy_(((torch.arange(n, device="cuda") * 3 + RANK + step) % 5 - 2).to(dtype))
        param.zero_()
        master.zero_()
        mom.zero_()
        torch.cuda.synchronize()
        if WORLD > 1:
            dist.barrier()
        for _ in range(3):
            a @ a                                   # fills every SM while the fused kernel's CTAs trickle in
        with torch.cuda.stream(side):
            comm.fused_allreduce_sgd(grad, param, master, mom, 1.0, 0.0, 0.0, zero_grads=True, nblocks=64, stream=side)
        torch.cuda.synchronize()
        want = sum(((torch.arange(n, device="cuda") * 3 + r + step) % 5 - 2).float() for r in range(WORLD)) / WORLD
        got = -param.float()                        # p = 0 - lr * mean(g), lr = 1, no momentum / decay
        bad = int((got != want.to(dtype).float()).sum())
        assert bad == 0, f"rank {RANK} step {step}: {bad} wrong elements (staggered CTAs corrupted the reduction)"
        assert int((grad != 0).sum()) == 0, "gradients were not re-zeroed"
    assert comm.status() == 0
    print(f"rank {RANK}: fused sgd with 64 staggered CTAs under a concurrent GEMM ok (world {WORLD})", flush=True)
    teardown()


def job_transport_ring():
    """All-reduce that rides the transport (parallel/transport_ring.py): ring over the plugin's connections, reduce-scatter
    hops are fused isends (the sender's kernel accumulates into the next rank's buffer over NVLink)."""
    from bagua_net_b200.parallel.transport_ring import TransportRing

    setup()
    ring = TransportRing()
    assert ring.transport == "nvl", ring.transport
    res = []
    for dtype, count in ((torch.float32, 1 << 20), (torch.bfloat16, 3 * (1 << 20) + 17), (torch.float32, 33), (torch.bfloat16, 32 << 20)):
        buf = ring.buffer(count, dtype)
        for rnd in range(2):
            buf.copy_(((torch.arange(count, device="cuda") * 5 + RANK + rnd) % 9 - 4).to(dtype))
            torch.cuda.synchronize()
            dist.barrier()
            ring.all_reduce(buf)
            want = sum(((torch.arange(count, device="cuda") * 5 + r + rnd) % 9 - 4).float() for r in range(WORLD))
            assert torch.equal(buf.float(), want), f"rank {RANK}: transport ring all-reduce {dtype} x{count} is wrong"
            dist.barrier()
        # bandwidth of the largest case
        if count >= (8 << 20):
            torch.cuda.synchronize()
            dist.barrier()
            t0 = time.perf_counter()
            iters = 5
            for _ in range(iters):
                ring.all_reduce(buf)
            dt = (time.perf_counter() - t0) / iters
            nbytes = count * buf.element_size()
            res.append((nbytes, nbytes / dt / 1e9 * 2 * (WORLD - 1) / WORLD))
    if RANK == 0:
        for nbytes, busbw in res:
            print(f"transport ring all-reduce {nbytes >> 20} MiB: busbw {busbw:.1f} GB/s (host-timed, world {WORLD}) stats {ring.core.stats()}",
                  flush=True)
    ring.close()
    teardown()


def job_transport_ring_compressed():
    """fp32 all-reduce with bf16 / fp8 on the wire (TransportRing.all_reduce_compressed): the quantisation rides the isend
    (fused) or runs as a local executor pass (unfused); every rank must end with the same bits."""
    from bagua_net_b200.parallel.transport_ring import TransportRing

    setup()
    ring = TransportRing()
    assert ring.transport == "nvl", ring.transport
    count = (4 << 20) + 1000
    buf = ring.buffer(count, torch.float32)
    gen = lambda r, rnd: (((torch.arange(count, device="cuda") * 7 + r * 3 + rnd) % 4) - 1).float() * 0.25   # noqa: E731
    for rnd, (wire, fused) in enumerate((("bf16", True), ("e4m3", True), ("e4m3", False), ("e5m2", True))):
        buf.copy_(gen(RANK, rnd))
        torch.cuda.synchronize()
        dist.barrier()
        ring.all_reduce_compressed(buf, wire=wire, scale=4.0, fused=fused)
        want = sum(gen(r, rnd) for r in range(WORLD))
        if wire == "e5m2":
            assert (buf - want).abs().max().item() <= 1.5
        else:
            assert torch.equal(buf, want), f"rank {RANK}: compressed all-reduce ({wire}, fused={fused}) is wrong"
        ref = buf.clone()
        dist.broadcast(ref, 0)
        assert torch.equal(ref, buf), f"rank {RANK}: ranks disagree after the compressed all-reduce ({wire})"
        st = ring.core.stats()
        wes = 2 if wire == "bf16" else 1
        assert st["bytes_sent"] <= 2 * (WORLD - 1) * (count // WORLD + 128) * wes, st
        dist.barrier()
    if RANK == 0:
        print(f"compressed transport-ring all-reduce ok (world {WORLD})", flush=True)
    ring.close()
    teardown()


def job_transport_mesh():
    """One-shot all-reduce over a full mesh of plugin connections (TransportMesh): one network step, the senders' kernels
    accumulate into every peer's output over NVLink."""
    from bagua_net_b200.parallel.transport_ring import TransportMesh

    setup()
    mesh = TransportMesh()
    assert mesh.transport == "nvl", mesh.transport
    res = []
    for idt, odt, count in ((torch.float32, torch.float32, 1 << 18), (torch.bfloat16, torch.float32, (1 << 20) + 24),
                            (torch.bfloat16, torch.bfloat16, 4096), (torch.float32, torch.float32, 9)):
        x, y = mesh.buffers(count, idt, odt)
        for rnd in range(2):
            x.copy_(((torch.arange(count, device="cuda") * 5 + RANK + rnd) % 9 - 4).to(idt))
            y.fill_(99)
            torch.cuda.synchronize()
            dist.barrier()
            mesh.all_reduce(x, y)
            want = sum(((torch.arange(count, device="cuda") * 5 + r + rnd) % 9 - 4).float() for r in range(WORLD))
            assert torch.equal(y.float(), want), f"rank {RANK}: mesh all-reduce {idt}->{odt} x{count} is wrong"
            dist.barrier()
        if count >= (1 << 18):
            torch.cuda.synchronize()
            dist.barrier()
            t0 = time.perf_counter()
            iters = 10
            for _ in range(iters):
                mesh.all_reduce(x, y)
            res.append((count * x.element_size(), (time.perf_counter() - t0) / iters))
    if RANK == 0:
        for nbytes, dt in res:
            print(f"transport mesh one-shot all-reduce {nbytes >> 10} KiB: {dt * 1e6:.1f} us per call (host-timed, world {WORLD})", flush=True)
    mesh.close()
    teardown()


def job_transport_mesh_twoshot():
    """Two-shot all-reduce over the mesh (reduce-scatter by fused isend into the slice owner, all-gather by copy), out of
    place and in place; ranks must end with identical bits even for data whose sums round."""
    from bagua_net_b200.parallel.transport_ring import TransportMesh

    setup()
    mesh = TransportMesh()
    assert mesh.transport == "nvl", mesh.transport
    res = []
    for idt, odt, count in ((torch.float32, torch.float32, 1 << 22), (torch.bfloat16, torch.float32, (1 << 20) + 24),
                            (torch.bfloat16, torch.bfloat16, 4096), (torch.float32, torch.float32, 9)):
        x, y = mesh.buffers(count, idt, odt)
        for rnd in range(2):
            x.copy_(((torch.arange(count, device="cuda") * 5 + RANK + rnd) % 9 - 4).to(idt))
            y.fill_(99)
            torch.cuda.synchronize()
            dist.barrier()
            mesh.all_reduce(x, y, algo="two-shot")
            want = sum(((torch.arange(count, device="cuda") * 5 + r + rnd) % 9 - 4).float() for r in range(WORLD))
            assert torch.equal(y.float(), want), f"rank {RANK}: two-shot all-reduce {idt}->{odt} x{count} is wrong"
            dist.barrier()
        if count >= (1 << 20):
            torch.cuda.synchronize()
            dist.barrier()
            t0 = time.perf_counter()
            iters = 10
            for _ in range(iters):
                mesh.all_reduce(x, y, algo="two-shot")
            res.append((count * x.element_size(), (time.perf_counter() - t0) / iters))
    # in place, random floats: the sums round, yet every rank must hold the owner's bits
    g = mesh.buffer(1 << 20, torch.float32)
    torch.manual_seed(100 + RANK)
    g.copy_(torch.randn(1 << 20, device="cuda"))
    mine = g.clone()
    torch.cuda.synchronize()
    dist.barrier()
    mesh.all_reduce(g, g, algo="two-shot")
    ref = mine.clone()
    dist.all_reduce(ref)
    assert (g - ref).abs().max().item() < 1e-4 * WORLD, "in-place two-shot all-reduce differs from NCCL's sum"
    digest = torch.stack([g.double().sum(), g.double().abs().sum()])
    alld = [torch.zeros_like(digest) for _ in range(WORLD)]
    dist.all_gather(alld, digest)
    assert all(torch.equal(alld[0], d_) for d_ in alld), "ranks hold different bits after the two-shot all-reduce"
    if RANK == 0:
        for nbytes, dt in res:
            busbw = nbytes / dt / 1e9 * 2 * (WORLD - 1) / WORLD
            print(f"transport mesh two-shot all-reduce {nbytes >> 10} KiB: {dt * 1e6:.1f} us per call, {busbw:.1f} GB/s busbw "
                  f"(host-timed, world {WORLD})", flush=True)
    mesh.close()
    teardown()


def job_tc_conv():
    from bagua_net_b200.ops import tc_conv, tc_linear

    setup()
    assert tc_linear.supported()
    assert tc_conv.self_check(verbose=RANK == 0), "wgmma convolution differs from cuDNN"
    print("wgmma conv3x3 forward + dgrad match cuDNN", flush=True)
    teardown()


def job_tc_conv_wgrad():
    """The wgmma filter gradient against cuDNN (several shapes, one and many pixel slices, scratch handed back clean),
    then inside a fused conv block: the autotuner may pick it per shape, training must look the same either way."""
    from bagua_net_b200.ops import tc_conv, tc_linear

    setup()
    assert tc_linear.supported()
    assert tc_conv.self_check_wgrad(verbose=RANK == 0), "wgmma filter gradient differs from cuDNN"
    os.environ["BNET_TC_WGRAD"] = "1"          # just checked in this very process
    x = torch.randn(8, 128, 28, 28, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    gy = torch.randn(8, 256, 28, 28, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last) / 28
    w = torch.randn(256, 128, 3, 3, device="cuda").bfloat16().contiguous(memory_format=torch.channels_last)
    ref = lambda: torch.ops.aten.convolution_backward(gy, x, w, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [False, True, False])[1]   # noqa: E731
    pick = tc_conv.choose_wgrad(gy, x, w, ref)
    print(f"wgmma conv3x3 filter gradient matches cuDNN; autotuner for 128->256 @28: {pick} {tc_conv.TIMINGS}", flush=True)
    teardown()


def job_grads_check():
    """bench.py's question before it relies on adopted gradients (BnetDDP writes them straight into the flat buffer): do they
    train like accumulated ones on this GPU?  Eager and captured; then the verdict of a deliberately broken hook."""
    from bagua_net_b200.parallel import ddp

    setup()
    os.environ.setdefault("BNET_TC_WGRAD", "0")      # (the filter-gradient kernel has a test of its own; no child process here)
    for graph in (False, True):
        ok, detail = ddp.direct_grads_self_check(torch.device("cuda", LOCAL), use_graph=graph)
        print(f"adopted vs accumulated gradients (cuda graph: {graph}): {ok} {detail}", flush=True)
        assert ok, detail
        assert detail["grad_copies_accumulate"] == 0
    real = ddp.BnetDDP._on_grad

    def lossy(self, p):
        if self._direct_grads and p.dim() == 4:
            p.grad = None
        return real(self, p)

    ddp.BnetDDP._on_grad = lossy
    ok, detail = ddp.direct_grads_self_check(torch.device("cuda", LOCAL), use_graph=False)
    ddp.BnetDDP._on_grad = real
    assert not ok, detail
    print(f"... and an engine that loses its filter gradients is rejected: {detail}", flush=True)
    teardown()


JOBS = {k[4:]: v for k, v in globals().items() if k.startswith("job_")}

if __name__ == "__main__":
    JOBS[sys.argv[1]]()

"""Per-rank bodies of the layout-free checkpoint GPU tests (launched by tests/test_checkpoint_reshard.py, one process per
GPU).  Usage: checkpoint_worker.py <job> <config> <dtype> <checkpoint path> [<second path>]."""
from __future__ import annotations

import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from adamw_worker import RANK, WORLD, same_on_every_rank, setup, teardown  # noqa: E402
from grad_accum_worker import ADAMW, SGD, TOL, global_batch, micro_grads, rel_updates, small_net  # noqa: E402
from lars_worker import LARS, larc_step  # noqa: E402

STEPS = 3                          # trained before the checkpoint, and again after it
# (engine keyword arguments, bucket_mb of the run that saves, bucket_mb of the run that resumes)
CONFIGS = {"sgd": (dict(optimizer="sgd", **SGD), 0.05, 0.02),
           "adamw-ema-groups": (dict(optimizer="adamw", **ADAMW, ema_decay=0.5), 0.05, 0.02),
           "lars-clip": (dict(optimizer="lars", **LARS, max_grad_norm=0.5), 0.02, 0.05)}
DTYPES = {"bf16": torch.bfloat16, "fp32": torch.float32}


def bits(t):
    return t.reshape(-1).contiguous().view(torch.uint8)


def same_state(a, b, path="state"):
    """Equal dicts, lists and numbers; tensors of the same dtype, shape, strides and bits."""
    assert type(a) is type(b), path
    if isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and a.shape == b.shape and a.stride() == b.stride(), path
        assert torch.equal(bits(a), bits(b)), f"{path}: bits differ"
    elif isinstance(a, dict):
        assert list(a) == list(b), path
        for k in a:
            same_state(a[k], b[k], f"{path}[{k!r}]")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            same_state(x, y, f"{path}[{i}]")
    else:
        assert a == b, f"{path}: {a!r} != {b!r}"


def deterministic():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False


def engine(comm, config, dtype, bucket_mb):
    from bagua_net_b200.parallel import BnetDDP, no_weight_decay_groups

    kw, _, _ = CONFIGS[config]
    torch.manual_seed(0)
    model = small_net().cuda().to(dtype).to(memory_format=torch.channels_last)
    groups = no_weight_decay_groups(model) if config.startswith("adamw") else None
    eng = BnetDDP(model, bucket_mb=bucket_mb, comm=comm, param_groups=groups, **kw)
    return model, eng


def release(eng):
    for h in eng._hooks:
        h.remove()


def train(eng, dtype, a, b):
    for step in range(a, b):
        xs, ys = global_batch(step)
        eng.train_step(xs[RANK].to(dtype).contiguous(memory_format=torch.channels_last), ys[RANK])
    torch.cuda.synchronize()


def save(model, eng, path):
    """Collective: rank 0 writes {"model", "optimizer"}; every rank returns once the file is complete."""
    full = eng.full_optimizer_state_dict()
    assert (full is None) == (RANK != 0)
    if RANK == 0:
        torch.save({"model": model.state_dict(), "optimizer": full}, path)
    if WORLD > 1:
        dist.barrier()
    return full


def load(model, eng, path):
    ck = torch.load(path, map_location="cpu")
    model.load_state_dict(ck["model"])
    eng.load_full_optimizer_state_dict(ck["optimizer"])
    return ck


def job_save(config, dtype, path):
    """Train STEPS steps at this world size and save."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    deterministic()
    comm = SymmComm(256 << 20)
    model, eng = engine(comm, config, DTYPES[dtype], CONFIGS[config][1])
    train(eng, DTYPES[dtype], 0, STEPS)
    save(model, eng, path)
    assert comm.status() == 0
    print(f"rank {RANK}: {config} {dtype}: {STEPS} steps at world {WORLD} ({len(eng.buckets)} buckets) saved", flush=True)
    teardown()


def _torch_reference(eng, model, ck, config):
    """A float64 copy of the model at the checkpoint's fp32 master weights, and torch.optim (SGD for LARS, which larc_step
    wraps) built from the engine's groups and loaded from the checkpoint's optimizer state."""
    state = ck["optimizer"]
    order = eng._torch_order()
    ref = small_net().cuda().double()
    rp = list(ref.parameters())
    with torch.no_grad():
        for i, j in enumerate(order):
            rp[j].copy_(state["bnet"]["master"][i])
    groups = [{"params": [rp[order[i]] for i in g["params"]]} for g in state["param_groups"]]
    if config.startswith("adamw"):
        opt = torch.optim.AdamW(groups, lr=ADAMW["lr"])
    else:
        opt = torch.optim.SGD(groups, lr=1.0, momentum=0.9)
    opt.load_state_dict(state)
    if config.startswith("lars"):
        for g in opt.param_groups:                    # (LARC folds the weight decay into the gradient)
            g["weight_decay"] = 0.0
    return ref, opt


def job_resume(config, dtype, path, path2):
    """Load at this world size (and the other bucket_mb), save again: bitwise the same dict.  Then STEPS more steps against
    a float64 torch.optim continuation from the same dict."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    deterministic()
    dt = DTYPES[dtype]
    comm = SymmComm(256 << 20)
    model, eng = engine(comm, config, dt, CONFIGS[config][2])
    ck = load(model, eng, path)
    full = save(model, eng, path2)
    if RANK == 0:
        same_state(full, ck["optimizer"])
    ref, opt = _torch_reference(eng, model, ck, config)
    p0 = [p.detach().clone() for p in ref.parameters()]
    probe = small_net().cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
    max_norm = CONFIGS[config][0].get("max_grad_norm")
    for step in range(STEPS, 2 * STEPS):
        xs, ys = global_batch(step)
        opt.zero_grad()
        if dt == torch.float32:
            torch.nn.functional.cross_entropy(ref(torch.cat(xs).double()), torch.cat(ys)).backward()
        else:
            micro_grads(model, probe, ref, xs, ys, 1)
        eng.train_step(xs[RANK].to(dt).contiguous(memory_format=torch.channels_last), ys[RANK])
        if max_norm is not None:
            torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm)
        if config.startswith("lars"):
            larc_step(list(ref.parameters()), opt)
        else:
            opt.step()
    torch.cuda.synchronize()
    total, worst = rel_updates(eng, model, ref, p0)
    tol_total, tol_worst, _ = TOL[dt]
    tag = f"{config} {dtype} resumed at world {WORLD}"
    assert total < tol_total and worst < tol_worst, f"{tag}: updates differ from float64 torch.optim: {total:.2e} / {worst:.2e}"
    assert same_on_every_rank(eng.flat_param), f"{tag}: ranks hold different parameters"
    assert comm.status() == 0
    print(f"rank {RANK}: {tag} ({len(eng.buckets)} buckets): re-saved dict bitwise equal; rel L2 of {STEPS} updates vs "
          f"float64 torch.optim {total:.2e} total, {worst:.2e} worst bucket", flush=True)
    teardown()


def job_exact(config, dtype, path):
    """At this world size and bucket_mb, 2 * STEPS steps in one run, and STEPS steps + save + load into a new engine + STEPS
    steps, are bitwise the same, eager and under a CUDA graph."""
    from bagua_net_b200.parallel import SymmComm

    setup()
    deterministic()
    dt = DTYPES[dtype]
    comm = SymmComm(256 << 20)
    bucket_mb = CONFIGS[config][1]
    for graph in (False, True):
        model, eng = engine(comm, config, dt, bucket_mb)
        eng.enable_cuda_graph(graph)
        train(eng, dt, 0, 2 * STEPS)
        want = [t.clone() for b in eng.buckets for t in b.state + ((b.ema,) if b.ema is not None else ())]
        want_p = eng.flat_param.clone()
        release(eng)
        model, eng = engine(comm, config, dt, bucket_mb)
        eng.enable_cuda_graph(graph)
        train(eng, dt, 0, STEPS)
        save(model, eng, path)
        release(eng)
        model, eng = engine(comm, config, dt, bucket_mb)
        eng.enable_cuda_graph(graph)
        load(model, eng, path)
        train(eng, dt, STEPS, 2 * STEPS)
        got = [t for b in eng.buckets for t in b.state + ((b.ema,) if b.ema is not None else ())]
        assert all(torch.equal(bits(a), bits(b)) for a, b in zip(got, want)), f"{config} graph={graph}: resumed state differs"
        assert torch.equal(bits(eng.flat_param), bits(want_p)), f"{config} graph={graph}: resumed parameters differ"
        release(eng)
        if WORLD > 1:
            dist.barrier()
    assert comm.status() == 0
    print(f"rank {RANK}: {config} {dtype}: resumed run bitwise the uninterrupted one at world {WORLD}, eager and graph",
          flush=True)
    teardown()


JOBS = {k[4:]: v for k, v in globals().items() if k.startswith("job_")}

if __name__ == "__main__":
    JOBS[sys.argv[1]](*sys.argv[2:])

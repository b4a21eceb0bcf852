"""The fused all-reduce + SGD kernel and the engine's SGD path on the GPU: the one-kernel step against float64 (bf16 and
fp32, four hyper-parameter sets, learning-rate changes, sizes at and around the ends of the kernel's 2-vector loop and
its tail for every grid size, guard regions, both entry points), NaN / Inf gradients against torch.optim.SGD, the
clipped step's apply stage against float64, and BnetDDP(optimizer="sgd") against torch.optim.SGD (+ clip_grad_norm_)
in eager and CUDA-graph mode with a checkpoint resumed mid-run.  The jobs are tests/sgd_worker.py; every job runs in
child processes, one per GPU."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "sgd_worker.py")


def _run(name, nproc=1, env=None, timeout=600):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    procs = []
    for r in range(nproc):
        e = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE=str(nproc), MASTER_ADDR="127.0.0.1",
                 MASTER_PORT=str(port), PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
        e.update(env or {})
        procs.append(subprocess.Popen([sys.executable, WORKER, name], env=e, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                                      text=True))
    outs = []
    for p in procs:
        try:
            o, err = p.communicate(timeout=timeout)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append((p.returncode, o, err))
    for rc, o, err in outs:
        print(o)
        assert rc == 0, f"job {name} failed rc={rc}\nstdout:\n{o[-4000:]}\nstderr:\n{err[-4000:]}"


def test_fused_sgd_kernel_matches_float64():
    _run("kernel")


def test_fused_sgd_nonfinite_gradients_match_torch_sgd():
    _run("nonfinite")


def test_clip_apply_sgd_matches_float64():
    _run("clip_apply")


def test_engine_sgd_matches_torch_sgd():
    _run("engine", timeout=900)


# Two GPUs: peer loads and stores.  (The in-switch path is chosen from three ranks on, where it beats the direct exchange.)
@pytest.mark.multigpu
@pytest.mark.parametrize("env", [{}, {"BNET_FUSED_NVLS": "0"}], ids=["auto", "p2p"])
@pytest.mark.parametrize("job", ["kernel", "nonfinite", "clip_apply", "engine"])
def test_fused_sgd_2gpu(job, env):
    _run(job, nproc=2, env=env, timeout=900)

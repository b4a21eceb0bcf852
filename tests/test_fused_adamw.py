"""The fused all-reduce + AdamW kernel and the engine's AdamW path on the GPU: the kernel against float64 (bf16 and fp32,
learning-rate changes, a step count of 10^5, every grid size, guard regions, NaN / Inf gradients against
torch.optim.AdamW), the CTA-paired gradient zeroing under staggered CTAs, and BnetDDP(optimizer="adamw") against
torch.optim.AdamW in eager and CUDA-graph mode with a checkpoint resumed mid-run.  The jobs are tests/adamw_worker.py;
every job runs in child processes, one per GPU."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "adamw_worker.py")


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


def test_fused_adamw_kernel_matches_float64():
    _run("kernel")


def test_fused_adamw_with_staggered_ctas():
    _run("staggered", timeout=240)


def test_engine_adamw_matches_torch_adamw():
    _run("engine", timeout=900)


# Two GPUs: peer loads and stores.  (The in-switch path is chosen from three ranks on, where it beats the direct exchange.)
@pytest.mark.multigpu
@pytest.mark.parametrize("env", [{}, {"BNET_FUSED_NVLS": "0"}], ids=["auto", "p2p"])
@pytest.mark.parametrize("job", ["kernel", "staggered", "engine"])
def test_fused_adamw_2gpu(job, env):
    _run(job, nproc=2, env=env, timeout=900)

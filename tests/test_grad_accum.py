"""Gradient accumulation in the fused data-parallel step, on the GPU: the accumulating reduce-and-norm stage against
float64 (guard regions, the partial row, the same bits for every grid size, re-zeroed gradients, the store-only stage
from a zeroed scratch), and BnetDDP(accumulation_steps=k) against a float64 torch.optim.SGD / AdamW (+ clip_grad_norm_)
on the global batch in eager and CUDA-graph mode.  The jobs are tests/grad_accum_worker.py; every job runs in child
processes, one per GPU."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "grad_accum_worker.py")


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


@pytest.mark.parametrize("job", ["kernel", "engine"])
def test_grad_accum(job):
    _run(job, timeout=900)


@pytest.mark.multigpu
@pytest.mark.parametrize("env", [{}, {"BNET_FUSED_NVLS": "0"}], ids=["auto", "p2p"])
@pytest.mark.parametrize("job", ["kernel", "engine"])
def test_grad_accum_2gpu(job, env):
    _run(job, nproc=2, env=env, timeout=900)

"""LARS in the fused data-parallel step, on the GPU: the per-chunk norm pass against float64 (world-2 and world-8
segment tables, guard regions, repeatable bits for every grid), the trust kernel (exclusion, zero norms, NaN and +-Inf,
the clip coefficient, the same bits on every rank), the apply stage against float64 per-tensor SGD (loop tails, every
grid) and BnetDDP(optimizer="lars") against a float64 LARC + torch.optim.SGD reference in eager and CUDA-graph mode.
The jobs are tests/lars_worker.py; every job runs in child processes, one per GPU."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "lars_worker.py")


def _run(name, nproc=1, env=None, timeout=900):
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


@pytest.mark.parametrize("job", ["norm", "trust", "apply", "engine"])
def test_fused_lars(job):
    _run(job)


@pytest.mark.multigpu
@pytest.mark.parametrize("env", [{}, {"BNET_FUSED_NVLS": "0"}], ids=["auto", "p2p"])
@pytest.mark.parametrize("job", ["norm", "trust", "apply", "engine"])
def test_fused_lars_2gpu(job, env):
    _run(job, nproc=2, env=env)

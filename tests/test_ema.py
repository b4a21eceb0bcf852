"""The exponential moving average of the master weights, on the GPU: the update kernel against float64 (loop tails for
1, 7, 132 and 264 CTAs, guard regions, NaN and +-Inf, the same bits for every grid, the copy and the skipped step) and
the advance kernel, and BnetDDP(ema_decay=...) against a float64 torch.optim + AveragedModel reference with SGD, AdamW
and LARS, f32 and bf16, eager and CUDA-graph mode, ema_every 1 and 2, k = 1 and 2, ema_parameters() included.  The jobs
are tests/ema_worker.py; every job runs in child processes, one per GPU."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "ema_worker.py")


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


@pytest.mark.parametrize("job", ["update", "engine"])
def test_ema(job):
    _run(job)


@pytest.mark.multigpu
@pytest.mark.parametrize("env", [{}, {"BNET_FUSED_NVLS": "0"}], ids=["auto", "p2p"])
@pytest.mark.parametrize("job", ["update", "engine"])
def test_ema_2gpu(job, env):
    _run(job, nproc=2, env=env)

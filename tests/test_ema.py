"""The exponential moving average of the master weights, on the GPU: the update kernel against float64 (loop tails for
1, 7, 132 and 264 CTAs, guard regions, NaN and +-Inf, the same bits for every grid, the copy and the skipped step) and
the advance kernel, and BnetDDP(ema_decay=...) against a float64 torch.optim + AveragedModel reference with SGD, AdamW
and LARS, f32 and bf16, eager and CUDA-graph mode, ema_every 1 and 2, k = 1 and 2, ema_parameters() included.  The jobs
are tests/ema_worker.py; every job runs in child processes, one per GPU."""
import os

import pytest
from gpu_jobs import run_ranks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "ema_worker.py")


@pytest.mark.parametrize("job", ["update", "engine"])
def test_ema(job):
    run_ranks(WORKER, [job], timeout=900)


@pytest.mark.multigpu
@pytest.mark.parametrize("env", [{}, {"BNET_FUSED_NVLS": "0"}], ids=["auto", "p2p"])
@pytest.mark.parametrize("job", ["update", "engine"])
def test_ema_2gpu(job, env):
    run_ranks(WORKER, [job], nproc=2, env=env, timeout=900)

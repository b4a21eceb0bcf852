"""LARS in the fused data-parallel step, on the GPU: the per-chunk norm pass against float64 (world-2 and world-8
segment tables, guard regions, repeatable bits for every grid), the trust kernel (exclusion, zero norms, NaN and +-Inf,
the clip coefficient, the same bits on every rank), the apply stage against float64 per-tensor SGD (loop tails, every
grid) and BnetDDP(optimizer="lars") against a float64 LARC + torch.optim.SGD reference in eager and CUDA-graph mode.
The jobs are tests/lars_worker.py; every job runs in child processes, one per GPU."""
import os

import pytest
from gpu_jobs import run_ranks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "lars_worker.py")


@pytest.mark.parametrize("job", ["norm", "trust", "apply", "engine"])
def test_fused_lars(job):
    run_ranks(WORKER, [job], timeout=900)


@pytest.mark.multigpu
@pytest.mark.parametrize("env", [{}, {"BNET_FUSED_NVLS": "0"}], ids=["auto", "p2p"])
@pytest.mark.parametrize("job", ["norm", "trust", "apply", "engine"])
def test_fused_lars_2gpu(job, env):
    run_ranks(WORKER, [job], nproc=2, env=env, timeout=900)

"""Parameter groups in the fused data-parallel step, on the GPU: the grouped one-kernel and apply-stage SGD and AdamW
kernels against the ungrouped kernels run per group, bitwise (loop tails, every grid, a group change at every tensor,
guard regions, clip coefficients 0.3 / 1e-3 / 1 / 0 / NaN), and BnetDDP(param_groups=...) against torch.optim with the same
groups in eager and CUDA-graph mode, with set_lr / set_param_group under a graph, clipping, accumulation, the EMA and a
checkpoint resumed mid-run.  The jobs are tests/param_groups_worker.py; every job runs in child processes, one per GPU."""
import os

import pytest
from gpu_jobs import run_ranks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "param_groups_worker.py")


@pytest.mark.parametrize("job", ["kernel", "apply", "engine"])
def test_param_groups(job):
    run_ranks(WORKER, [job], timeout=900)


@pytest.mark.multigpu
@pytest.mark.parametrize("env", [{}, {"BNET_FUSED_NVLS": "0"}], ids=["auto", "p2p"])
@pytest.mark.parametrize("job", ["kernel", "apply", "engine"])
def test_param_groups_2gpu(job, env):
    run_ranks(WORKER, [job], nproc=2, env=env, timeout=900)

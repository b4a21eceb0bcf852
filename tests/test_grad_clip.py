"""Gradient clipping by global norm in the fused data-parallel step, on the GPU: the reduce-and-square-norm stage against
float64 (every grid size, guard regions, repeatable bits, re-zeroed gradients), the norm and coefficient against
torch.nn.utils.clip_grad_norm_ (thresholds below, at and above the norm, zero and non-finite gradients), bitwise identity
with the one-kernel step at max_norm = inf, the CTA-paired zeroing under staggered CTAs, and BnetDDP(max_grad_norm=...)
against torch.optim.AdamW + clip_grad_norm_ in eager and CUDA-graph mode.  The jobs are tests/grad_clip_worker.py; every
job runs in child processes, one per GPU."""
import os

import pytest
from gpu_jobs import run_ranks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "grad_clip_worker.py")


@pytest.mark.parametrize("job", ["kernel", "coef", "identity", "staggered", "engine"])
def test_grad_clip(job):
    run_ranks(WORKER, [job], timeout=900)


@pytest.mark.multigpu
@pytest.mark.parametrize("env", [{}, {"BNET_FUSED_NVLS": "0"}], ids=["auto", "p2p"])
@pytest.mark.parametrize("job", ["kernel", "coef", "identity", "staggered", "engine"])
def test_grad_clip_2gpu(job, env):
    run_ranks(WORKER, [job], nproc=2, env=env, timeout=900)

"""Gradient accumulation in the fused data-parallel step, on the GPU: the accumulating reduce-and-norm stage against
float64 (guard regions, the partial row, the same bits for every grid size, re-zeroed gradients, the store-only stage
from a zeroed scratch), and BnetDDP(accumulation_steps=k) against a float64 torch.optim.SGD / AdamW (+ clip_grad_norm_)
on the global batch in eager and CUDA-graph mode.  The jobs are tests/grad_accum_worker.py; every job runs in child
processes, one per GPU."""
import os

import pytest
from gpu_jobs import run_ranks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "grad_accum_worker.py")


@pytest.mark.parametrize("job", ["kernel", "engine"])
def test_grad_accum(job):
    run_ranks(WORKER, [job], timeout=900)


@pytest.mark.multigpu
@pytest.mark.parametrize("env", [{}, {"BNET_FUSED_NVLS": "0"}], ids=["auto", "p2p"])
@pytest.mark.parametrize("job", ["kernel", "engine"])
def test_grad_accum_2gpu(job, env):
    run_ranks(WORKER, [job], nproc=2, env=env, timeout=900)

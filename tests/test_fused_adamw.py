"""The fused all-reduce + AdamW kernel and the engine's AdamW path on the GPU: the kernel against float64 (bf16 and fp32,
learning-rate changes, a step count of 10^5, every grid size, guard regions, NaN / Inf gradients against
torch.optim.AdamW), the CTA-paired gradient zeroing under staggered CTAs, and BnetDDP(optimizer="adamw") against
torch.optim.AdamW in eager and CUDA-graph mode with a checkpoint resumed mid-run.  The jobs are tests/adamw_worker.py;
every job runs in child processes, one per GPU."""
import os

import pytest
from gpu_jobs import run_ranks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "adamw_worker.py")


def test_fused_adamw_kernel_matches_float64():
    run_ranks(WORKER, ["kernel"])


def test_fused_adamw_with_staggered_ctas():
    run_ranks(WORKER, ["staggered"], timeout=240)


def test_engine_adamw_matches_torch_adamw():
    run_ranks(WORKER, ["engine"], timeout=900)


# Two GPUs: peer loads and stores.  (The in-switch path is chosen from three ranks on, where it beats the direct exchange.)
@pytest.mark.multigpu
@pytest.mark.parametrize("env", [{}, {"BNET_FUSED_NVLS": "0"}], ids=["auto", "p2p"])
@pytest.mark.parametrize("job", ["kernel", "staggered", "engine"])
def test_fused_adamw_2gpu(job, env):
    run_ranks(WORKER, [job], nproc=2, env=env, timeout=900)

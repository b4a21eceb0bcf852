"""The fused all-reduce + SGD kernel and the engine's SGD path on the GPU: the one-kernel step against float64 (bf16 and
fp32, four hyper-parameter sets, learning-rate changes, sizes at and around the ends of the kernel's 2-vector loop and
its tail for every grid size, guard regions, both entry points), NaN / Inf gradients against torch.optim.SGD, the
clipped step's apply stage against float64, and BnetDDP(optimizer="sgd") against torch.optim.SGD (+ clip_grad_norm_)
in eager and CUDA-graph mode with a checkpoint resumed mid-run.  The jobs are tests/sgd_worker.py; every job runs in
child processes, one per GPU."""
import os

import pytest
from gpu_jobs import run_ranks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "sgd_worker.py")


def test_fused_sgd_kernel_matches_float64():
    run_ranks(WORKER, ["kernel"])


def test_fused_sgd_nonfinite_gradients_match_torch_sgd():
    run_ranks(WORKER, ["nonfinite"])


def test_clip_apply_sgd_matches_float64():
    run_ranks(WORKER, ["clip_apply"])


def test_engine_sgd_matches_torch_sgd():
    run_ranks(WORKER, ["engine"], timeout=900)


# Two GPUs: peer loads and stores.  (The in-switch path is chosen from three ranks on, where it beats the direct exchange.)
@pytest.mark.multigpu
@pytest.mark.parametrize("env", [{}, {"BNET_FUSED_NVLS": "0"}], ids=["auto", "p2p"])
@pytest.mark.parametrize("job", ["kernel", "nonfinite", "clip_apply", "engine"])
def test_fused_sgd_2gpu(job, env):
    run_ranks(WORKER, [job], nproc=2, env=env, timeout=900)

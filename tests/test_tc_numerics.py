"""The wgmma linear / convolution kernels in every tile configuration against float64 (exact on integer data, within the
bf16 + fp32 rounding bound on Gaussian data), and NaN / Inf through the fused epilogues and layers against eager torch.
The cases and the jobs are tests/tc_numerics_worker.py; every GPU job runs in a child process."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "tc_numerics_worker.py")


def _job(name, timeout=600, env=None):
    e = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    e.update(env or {})
    out = subprocess.run([sys.executable, WORKER, name], env=e, capture_output=True, text=True, timeout=timeout)
    print(out.stdout)
    assert out.returncode == 0, f"job {name} failed rc={out.returncode}\nstdout:\n{out.stdout[-4000:]}\nstderr:\n{out.stderr[-4000:]}"
    return out.stdout


def test_case_list_reaches_every_instantiation():
    """With the host planner's 132-SM default: every instantiation is reached and every tile width runs persistent once, so
    a planner change that moves a case off its target fails here, without a GPU."""
    _job("coverage", timeout=120, env={"CUDA_VISIBLE_DEVICES": ""})


@pytest.mark.gpu
def test_case_list_reaches_every_instantiation_on_this_gpu():
    _job("coverage", timeout=120)


@pytest.mark.gpu
def test_linear_kernels_match_float64():
    _job("linear")


@pytest.mark.gpu
def test_conv_kernels_match_float64():
    _job("conv")


@pytest.mark.gpu
def test_vgg16_batch32_tilings_match_float64():
    _job("vgg", timeout=900)


@pytest.mark.gpu
def test_nan_and_inf_follow_eager_torch():
    _job("nan")


@pytest.mark.gpu
def test_fused_column_reductions_are_reproducible_with_shifted_bn_stats():
    """Bias-gradient and BatchNorm reductions give identical bits in three calls; the BatchNorm statistics are the sums of
    z - K and (z - K)^2 with K each channel's row-0 value."""
    _job("reductions")

"""The fused layer kernels (bias + ReLU, 2x2 max-pool, their backward passes and bias-gradient reductions, the BatchNorm
family) against float64 at every launch shape: channel widths that do and do not divide the block, row counts around the
block step and past the grid cap, guard bands around every output.  The cases and the jobs are tests/nn_numerics_worker.py;
every GPU job runs in a child process."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "nn_numerics_worker.py")


def _job(name, timeout=900, env=None):
    e = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    e.update(env or {})
    out = subprocess.run([sys.executable, WORKER, name], env=e, capture_output=True, text=True, timeout=timeout)
    print(out.stdout)
    assert out.returncode == 0, f"job {name} failed rc={out.returncode}\nstdout:\n{out.stdout[-4000:]}\nstderr:\n{out.stderr[-4000:]}"
    return out.stdout


# the reductions' grid cap: blocks per SM (the library's default is 2); it changes the grid and the number of partial rows
BLOCKS_PER_SM = ("2", "1", "16")


@pytest.mark.gpu
def test_bias_relu_and_pool_forward_are_exact():
    _job("elementwise")


@pytest.mark.gpu
@pytest.mark.parametrize("blocks_per_sm", BLOCKS_PER_SM)
def test_relu_and_pool_backward_match_float64(blocks_per_sm):
    _job("backward", env={"BNET_NN_BLOCKS_PER_SM": blocks_per_sm})


@pytest.mark.gpu
@pytest.mark.parametrize("blocks_per_sm", BLOCKS_PER_SM)
def test_batchnorm_kernels_match_float64(blocks_per_sm):
    _job("batchnorm", env={"BNET_NN_BLOCKS_PER_SM": blocks_per_sm})


@pytest.mark.gpu
def test_batchnorm_non_finite_values_follow_eager_torch():
    _job("nonfinite")


@pytest.mark.gpu
def test_layers_wider_than_the_kernels_fall_back_to_eager():
    _job("layer_gate")

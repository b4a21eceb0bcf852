"""The fused-step kernel jobs at three ranks and at eight (or the most GPUs the machine has, if that is four to seven),
on both paths.  The one- and two-GPU tests of the other files never reach the in-switch (NVLS) step, which the kernels
take from three ranks on, nor the peer-load bodies used above two ranks:

* W = 3, auto: NVLS at an odd world size;        W = 3, p2p: the generic (not unrolled) peer-load reduction;
* W = 8, auto: what the benchmark runs;          W = 8, p2p: the unrolled eight-rank peer-load body.

`BNET_FUSED_NVLS=0` forces the peer-load path.  Without multicast the auto cases would quietly run the p2p path again, so
they skip instead, saying why; a probe job reads `SymmComm.has_multicast` once per world size."""
import os

import pytest
from gpu_jobs import run_ranks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATHS = [pytest.param({}, id="auto"), pytest.param({"BNET_FUSED_NVLS": "0"}, id="p2p")]


def _gpus():
    try:
        import torch

        return torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        return 0


def _big_world():
    """8, or the machine's GPU count when it has four to seven (fewer: 8, and the cases skip)."""
    n = _gpus()
    return n if 4 <= n < 8 else 8


WORLDS = [3, _big_world()]
_MULTICAST = {}


def has_multicast(world):
    """Whether a `world`-rank SymmComm binds a multicast object on this machine (one probe job per world size)."""
    if world not in _MULTICAST:
        outs = run_ranks(os.path.join(ROOT, "tests", "allreduce_worker.py"), ["probe"], nproc=world, timeout=300)
        _MULTICAST[world] = "multicast=True" in outs[0][1]
    return _MULTICAST[world]


def run_at(world, worker, job, env, timeout=900):
    if _gpus() < world:
        pytest.skip(f"world size {world} needs {world} GPUs; this machine has {_gpus()}")
    if not env and not has_multicast(world):
        pytest.skip(f"no multicast at world size {world}: the auto path would be the p2p path again")
    run_ranks(os.path.join(ROOT, "tests", worker), [job], nproc=world, env=env, timeout=timeout)


JOBS = [("sgd_worker.py", j) for j in ("kernel", "nonfinite", "clip_apply")] + \
       [("adamw_worker.py", j) for j in ("kernel", "staggered")] + \
       [("grad_clip_worker.py", j) for j in ("kernel", "coef", "identity", "staggered")] + \
       [("grad_accum_worker.py", "kernel")] + \
       [("lars_worker.py", j) for j in ("norm", "trust", "apply")] + \
       [("param_groups_worker.py", j) for j in ("kernel", "apply")] + \
       [("gpu_worker.py", "fused_sgd_staggered")]


@pytest.mark.parametrize("env", PATHS)
@pytest.mark.parametrize("world", WORLDS, ids=lambda w: f"w{w}")
@pytest.mark.parametrize("worker,job", JOBS, ids=[f"{w[:-10]}-{j}" for w, j in JOBS])
def test_fused_job_at_world_size(worker, job, world, env):
    run_at(world, worker, job, env)


def test_engine_sgd_at_largest_world_size_auto():
    """BnetDDP(optimizer="sgd") against torch.optim.SGD in the benchmark's configuration: every rank, the default path."""
    run_at(WORLDS[-1], "sgd_worker.py", "engine", {}, timeout=1200)

"""The symmetric-heap all-reduce kernels against float64 at every world size: two-shot peer loads/stores, the in-switch
(NVLS) kernel when the machine has multicast, the one-shot kernel and the barrier-free LL kernel, for f32 / bf16 / f16
and sum / avg / max / min.  Element-wise fp32 error bounds, guard regions on every rank, the same bits on every rank and
for every grid size, loop-tail sizes of the body each world size runs, NaN / Inf inputs against float64 and NCCL, and
the multi-tensor pack + cast kernel.  The jobs are tests/allreduce_worker.py, one process per GPU; a world size above
the machine's GPU count skips."""
import os

import pytest
from gpu_jobs import run_ranks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "allreduce_worker.py")


def _gpus():
    try:
        import torch

        return torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        return 0


# 2, 3 (a 1/W that is not exact, the generic peer-load loop), 4, 8 (the unrolled bodies), and the machine's own GPU count
WORLDS = sorted({2, 3, 4, 8} | ({_gpus()} if 1 <= _gpus() <= 8 else set()))


def run_at(world, job, timeout=900):
    if _gpus() < world:
        pytest.skip(f"world size {world} needs {world} GPUs; this machine has {_gpus()}")
    run_ranks(WORKER, [job], nproc=world, timeout=timeout)


@pytest.mark.parametrize("world", WORLDS, ids=lambda w: f"w{w}")
@pytest.mark.parametrize("job", ["twoshot", "oneshot", "ll", "nonfinite"])
def test_allreduce_matches_float64(job, world):
    run_at(world, job)


def test_pack_cast_all_dtype_pairs():
    run_at(1, "pack_cast")

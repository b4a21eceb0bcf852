"""The layout-free optimizer state on the GPU: saved at one world size and loaded at another (and another bucket_mb), saved
again bitwise the same, and trained on as a float64 torch.optim continuation from the same dict (Apex LARC for LARS);
resumed at the same world size and bucket_mb, bitwise the uninterrupted run, eager and under a CUDA graph; and the VGG16
example saving at one world size and resuming at another.  The jobs are tests/checkpoint_worker.py, one process per GPU;
world sizes the machine has not the GPUs for are skipped."""
import os

import pytest
from gpu_jobs import run_ranks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "checkpoint_worker.py")
# (config, model dtype): one bf16 and one fp32 model among them
CONFIGS = [("sgd", "bf16"), ("adamw-ema-groups", "fp32"), ("lars-clip", "bf16")]


def _gpus():
    try:
        import torch

        return torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        return 0


def _need(world):
    if _gpus() < world:
        pytest.skip(f"world size {world} needs {world} GPUs; this machine has {_gpus()}")


@pytest.mark.parametrize("worlds", [(1, 1), (1, 2), (2, 1), (3, 8)], ids=lambda w: f"w{w[0]}-w{w[1]}")
@pytest.mark.parametrize("config,dtype", CONFIGS, ids=[f"{c}-{d}" for c, d in CONFIGS])
def test_reshard_round_trip_and_continuation(config, dtype, worlds, tmp_path):
    """(1, 1) changes only bucket_mb; the others the world size as well."""
    _need(max(worlds))
    a, b = str(tmp_path / "a.pt"), str(tmp_path / "b.pt")
    run_ranks(WORKER, ["save", config, dtype, a], nproc=worlds[0], timeout=900)
    run_ranks(WORKER, ["resume", config, dtype, a, b], nproc=worlds[1], timeout=900)


@pytest.mark.parametrize("world", [1, 2], ids=lambda w: f"w{w}")
@pytest.mark.parametrize("config,dtype", CONFIGS, ids=[f"{c}-{d}" for c, d in CONFIGS])
def test_resume_at_same_world_is_bitwise(config, dtype, world, tmp_path):
    _need(world)
    run_ranks(WORKER, ["exact", config, dtype, str(tmp_path / "ck.pt")], nproc=world, timeout=900)


@pytest.mark.parametrize("worlds", [(1, 1), (2, 1)], ids=lambda w: f"w{w[0]}-w{w[1]}")
def test_vgg16_example_saves_and_resumes(worlds, tmp_path):
    _need(max(worlds))
    example = os.path.join(ROOT, "examples", "train_vgg16.py")
    ck = str(tmp_path / "vgg16.pt")
    run_ranks(example, ["--steps", "3", "--batch", "8", "--ema-decay", "0.999", "--checkpoint", ck], nproc=worlds[0],
              timeout=900)
    assert os.path.exists(ck)
    outs = run_ranks(example, ["--steps", "3", "--batch", "8", "--ema-decay", "0.999", "--resume", ck], nproc=worlds[1],
                     timeout=900)
    assert "resumed from" in outs[0][1]

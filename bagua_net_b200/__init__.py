"""bagua_net_b200 — a Hopper-native NCCL network transport + fused collectives.

Python face of the native library ``libnccl-net.so`` (C++ engine, multi-stream TCP
transports, intra-host shared-memory/NVLink transport, sm_90a kernels):

* ``bagua_net_b200.utils``    — plugin loader, ctypes view of the ncclNet ABI tables,
  NIC discovery, telemetry readers, env helpers (what the reference exposes through
  environment variables only; reference: SURVEY.md §2.7).
* ``bagua_net_b200.ops``      — hand-written sm_90a collectives/fused ops (NVLS
  multimem all-reduce, P2P all-reduce, fused all-reduce+SGD, pack/cast).
* ``bagua_net_b200.parallel`` — symmetric-memory communicator and the DDP engine
  that rides on those kernels (the reference's consumer is PyTorch/Bagua DDP,
  reference README.md:52-84).
* ``bagua_net_b200.models``   — the benchmark model families (VGG16, ResNet-50).
"""
from __future__ import annotations

import os

__version__ = "0.2.0"

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
REPO_ROOT = os.path.dirname(_PKG_DIR)
# BNET_LIB_DIR points the loader at another build of the same library (sanitizer builds: `make tsan`).
LIB_DIR = os.environ.get("BNET_LIB_DIR") or os.path.join(_PKG_DIR, "lib")
LIB_NAME = "libnccl-net.so"


def lib_path(name: str = LIB_NAME) -> str:
    return os.path.join(LIB_DIR, name)


def build(verbose: bool = False, jobs: int | None = None) -> str:
    """Compile the native library in-tree (nvcc cross-compiles sm_90a without a GPU)."""
    from ._build import build_native

    return build_native(verbose=verbose, jobs=jobs)


def load_library(name: str = LIB_NAME):
    """ctypes handle of the native library; builds it on first use if it is missing."""
    from .utils.native import load

    return load(name)

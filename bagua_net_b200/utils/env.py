"""Environment helpers: how to make NCCL load the bnet plugin.

The reference documents one step — put the directory holding libnccl-net.so on
LD_LIBRARY_PATH and look for "NCCL INFO Using network BaguaNet" (reference
README.md:32-45).  Inside one NVSwitch box NCCL would never use a network plugin on
its own (it picks P2P/NVLS/SHM), so ``force_net`` also disables those transports —
that is how a net plugin is exercised on a single node.
"""
from __future__ import annotations

import os

from .. import LIB_DIR


# NCCL drives a net plugin through a proxy pipeline of NCCL_BUFFSIZE/8-byte slices per channel; with the default
# 4 MiB buffers and 2-4 channels that pipeline, not the link, bounds the throughput
TUNED = {"NCCL_BUFFSIZE": str(32 << 20), "NCCL_MIN_NCHANNELS": "16", "NCCL_PROTO": "Simple"}


def nccl_plugin_env(plugin: str = "bnet", force_net: bool = False, gdr: bool = True, debug: bool = False,
                    extra: dict | None = None, tuned: bool = False, eager_modules: bool = True) -> dict:
    """Environment variables (as a dict) that make NCCL >= 2.2x dlopen our plugin.

    plugin: "bnet" -> libnccl-net-bnet.so (tables v3..v8); "bnetx" adds the v9/v10 tables.
    """
    ld = os.environ.get("LD_LIBRARY_PATH", "")
    env = {
        "LD_LIBRARY_PATH": LIB_DIR + (os.pathsep + ld if ld else ""),
        "NCCL_NET_PLUGIN": plugin,
        "NCCL_NET": "BNet",
    }
    if os.environ.get("BNET_TUNER", "1") != "0" and plugin == "bnet":
        # protocol choice per message size over this transport (csrc/plugin/tuner.cc): libnccl-tuner-bnet.so
        env["NCCL_TUNER_PLUGIN"] = "bnet"
    if "CUDA_DEVICE_MAX_CONNECTIONS" not in os.environ:
        # the transport keeps up to 8 resident stream kernels, each on its own CUDA stream; with the default
        # of 8 hardware work queues per context other streams (NCCL's, the staging copies) can end up queued
        # BEHIND a resident kernel.  32 queues keep them independent.
        env["CUDA_DEVICE_MAX_CONNECTIONS"] = "32"
    if eager_modules and "CUDA_MODULE_LOADING" not in os.environ:
        # CUDA loads kernels lazily, and the first launch of a kernel waits for the device to drain.  If the APPLICATION
        # launches a kernel for the first time while a collective is in flight, that wait never ends: the NCCL kernel is
        # waiting for this transport's copy kernel, whose launch sits behind the loader (seen under torch DDP: the
        # proxy thread stuck inside cudaLaunchKernelEx).  Stock NCCL never launches from its
        # proxy, so it is immune; a transport that moves data with kernels needs every module loaded up front.
        # The price is start-up time (torch + cuDNN + cuBLAS hold gigabytes of kernels: 100 s per process measured with
        # 2 ranks, 260 s with 4).  eager_modules=False leaves loading lazy: then the APPLICATION has to launch each of
        # its kernels once while no collective is in flight (bench.py does: warm-up steps + a single-rank DDP dry run).
        env["CUDA_MODULE_LOADING"] = "EAGER"
    if force_net:
        env.update({"NCCL_P2P_DISABLE": "1", "NCCL_SHM_DISABLE": "1", "NCCL_NVLS_ENABLE": "0",
                    "NCCL_NET_DISABLE_INTRA": "0"})
    if gdr:
        # our "NIC" is the NVLink fabric: let NCCL hand us device pointers wherever the GPU sits
        env.update({"NCCL_NET_GDR_LEVEL": "SYS", "NCCL_NET_GDR_READ": "1", "NCCL_DMABUF_ENABLE": "0"})
    else:
        env["BNET_GDR"] = "0"
    if debug:
        env.update({"NCCL_DEBUG": "INFO", "NCCL_DEBUG_SUBSYS": "INIT,NET,ENV"})
    if tuned:
        env.update({k: v for k, v in TUNED.items() if k not in os.environ})
    if extra:
        env.update(extra)
    return env


def apply(env: dict) -> None:
    os.environ.update(env)


if __name__ == "__main__":   # `env $(python -m bagua_net_b200.utils.env) <cmd>` loads the plugin into NCCL
    import sys

    kw = {"force_net": "--no-force" not in sys.argv, "debug": "--debug" in sys.argv, "gdr": "--no-gdr" not in sys.argv,
          "tuned": "--tuned" in sys.argv}
    print(" ".join(f"{k}={v}" for k, v in nccl_plugin_env(**kw).items()))

"""`python -m bagua_net_b200.doctor` — check that this machine can run the plugin and print what to export.

The reference's only guidance is a README paragraph (set LD_LIBRARY_PATH, look for "Using network BaguaNet" in the
NCCL log: reference README.md:32-45).  This goes through the things that actually go wrong: the library builds and
loads, the tables NCCL will probe are exported, which NCCL is installed and which ABI version it will pick, the
interfaces NCCL_SOCKET_IFNAME selects, room in /dev/shm for the per-connection mailboxes, CUDA work queues, and —
on a GPU box — peer access and multicast (NVLS) support.
"""
from __future__ import annotations

import ctypes
import json
import os
import shutil
import sys


def _nccl_versions() -> list[str]:
    found = []
    try:
        import torch

        found.append("torch-bundled NCCL " + ".".join(str(x) for x in torch.cuda.nccl.version()))
    except Exception:
        pass
    for name in ("libnccl.so.2", "libnccl.so"):
        try:
            lib = ctypes.CDLL(name)
            v = ctypes.c_int()
            if lib.ncclGetVersion(ctypes.byref(v)) == 0:
                found.append(f"system {name} {v.value // 10000}.{v.value // 100 % 100}.{v.value % 100}")
                break
        except OSError:
            continue
    return found


def run(out=sys.stdout) -> int:
    import bagua_net_b200
    from bagua_net_b200.utils import native
    from bagua_net_b200.utils.env import nccl_plugin_env

    problems = 0

    def say(ok, what, detail=""):
        nonlocal problems
        if ok is False:
            problems += 1
        mark = {True: "ok  ", False: "FAIL", None: "note"}[ok]
        print(f"[{mark}] {what}" + (f": {detail}" if detail else ""), file=out)

    # 1. library and exported tables
    try:
        path = bagua_net_b200.build()
        lib = bagua_net_b200.load_library()
        say(True, "native library", f"{path} ({native.version()})")
    except Exception as e:          # noqa: BLE001 - report and stop: nothing else can be checked
        say(False, "native library", str(e))
        return 1
    have = []
    for v in range(3, 11):
        for name in (bagua_net_b200.LIB_NAME, "libnccl-net-bnetx.so"):
            try:
                ctypes.c_void_p.in_dll(bagua_net_b200.load_library(name), f"ncclNetPlugin_v{v}")
                have.append(f"v{v}" + ("" if name == bagua_net_b200.LIB_NAME else "(bnetx)"))
                break
            except (ValueError, OSError):
                continue
    say("v8" in have, "ncclNet tables exported", " ".join(have))
    coll = []
    for v in (4, 6, 7, 8, 9, 10):
        for name in (bagua_net_b200.LIB_NAME, "libnccl-net-bnetx.so"):
            try:
                ctypes.c_void_p.in_dll(bagua_net_b200.load_library(name), f"ncclCollNetPlugin_v{v}")
                coll.append(f"v{v}" + ("" if name == bagua_net_b200.LIB_NAME else "(bnetx)"))
                break
            except (ValueError, OSError):
                continue
    say("v8" in coll, "ncclCollNet tables exported", " ".join(coll) + (
        " — switched on (BNET_COLLNET=1): with NCCL_COLLNET_ENABLE=1 NCCL may offload all-reduces to the two-shot mesh"
        if os.environ.get("BNET_COLLNET") == "1" else " — silent (no devices reported) unless BNET_COLLNET=1"))
    for line in _nccl_versions() or ["no NCCL found (the plugin is still usable through bagua_net_b200.utils.abi)"]:
        say(None, "NCCL", line + " — NCCL 2.19+ probes v6..v10 tables; 2.6-2.18 load v4")
    del lib

    # 2. what the engine will do with the current environment
    cfg = native.config()
    say(True, "engine configuration", json.dumps({k: cfg[k] for k in sorted(cfg) if k in (
        "implement", "nstreams", "min_chunksize", "nvl", "gdr", "shm_ring_bytes", "timeout_ms")}))
    ifs = native.find_interfaces(os.environ.get("NCCL_SOCKET_IFNAME"))
    say(bool(ifs), "interfaces selected by NCCL_SOCKET_IFNAME=" + os.environ.get("NCCL_SOCKET_IFNAME", "(default ^docker,lo)"),
        ", ".join(f"{i.get('name')}[{i.get('addr', '?')}, {i.get('speed', '?')} Mb/s]" for i in ifs) or "none")

    # 3. /dev/shm: one mailbox (ring + descriptors) per same-host connection, dozens of connections per rank
    try:
        free = shutil.disk_usage("/dev/shm").free
        per = int(cfg.get("shm_ring_bytes", 1 << 20)) + (1 << 17)
        say(free > 64 * per, "/dev/shm", f"{free >> 20} MiB free, ~{per >> 10} KiB per same-host connection "
            f"(room for ~{free // per} connections; lower BNET_SHM_RING_BYTES or enlarge /dev/shm if this is small)")
    except OSError as e:
        say(None, "/dev/shm", str(e))

    # 4. CUDA side
    try:
        import torch

        ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        ngpu = 0
    if ngpu == 0:
        say(None, "CUDA", "no GPU visible: TCP and shared-memory transports only (the NVLink kernels need sm_90a)")
    else:
        import torch

        cap = torch.cuda.get_device_capability(0)
        say(tuple(cap) == (9, 0), "GPU", f"{ngpu} x {torch.cuda.get_device_name(0)} (sm_{cap[0]}{cap[1]}); kernels are built for sm_90a")
        if ngpu > 1:
            peer = all(torch.cuda.can_device_access_peer(0, j) for j in range(1, ngpu))
            say(peer, "peer access GPU0 -> others", "NVLink/PCIe P2P" if peer else "not available: the NVL direct path falls back to the staged ring")
        q = os.environ.get("CUDA_DEVICE_MAX_CONNECTIONS")
        say(None if q is None else int(q) >= 16, "CUDA_DEVICE_MAX_CONNECTIONS", (q or "unset (8)") +
            " — the transport keeps up to 8 resident kernels on their own streams; 32 keeps other streams independent")
        try:
            from bagua_net_b200.parallel import SymmComm

            c = SymmComm(4 << 20)           # cuMemCreate + export + map of a symmetric heap (single rank here)
            c.close()
            say(True, "symmetric heap (cuMem VMM, POSIX-fd exportable)")
        except Exception as e:      # noqa: BLE001
            say(False, "symmetric heap", str(e))
        try:
            from bagua_net_b200.ops import tc_conv

            v = tc_conv.prepare()
            say(None, "wgmma kernels", f"linear / convolution self-check {'passed' if v['usable'] else 'not passed (cuBLAS / cuDNN are used)'}; "
                f"filter gradient {'trusted' if v['wgrad'] else 'not trusted'} on this GPU"
                + (f" with {os.environ['BNET_TC_WGRAD_BN']}-column tiles" if v["wgrad"] and os.environ.get("BNET_TC_WGRAD_BN") else ""))
        except Exception as e:      # noqa: BLE001
            say(None, "wgmma kernels", f"could not be checked: {e}")
        try:
            cu = ctypes.CDLL("libcuda.so.1")
            dev, val = ctypes.c_int(), ctypes.c_int()
            cu.cuInit(0)
            cu.cuDeviceGet(ctypes.byref(dev), 0)
            CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED = 132
            ok = cu.cuDeviceGetAttribute(ctypes.byref(val), CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) == 0 and val.value == 1
            say(None, "multicast (NVLS) support", "yes: all-reduce reduces inside the NVSwitch for more than two ranks"
                if ok else "no: all-reduce uses the peer load/store kernels")
        except OSError as e:
            say(None, "multicast (NVLS) support", f"cannot query the driver: {e}")

    # 5. what to export
    env = nccl_plugin_env(force_net=False)
    print("\n# to make NCCL load the plugin:", file=out)
    print("export " + " ".join(f"{k}={v}" for k, v in env.items()), file=out)
    print("# inside ONE box NCCL only uses a net plugin when its own transports are off (benchmarking the plugin):", file=out)
    print("export NCCL_P2P_DISABLE=1 NCCL_SHM_DISABLE=1 NCCL_NVLS_ENABLE=0", file=out)
    from bagua_net_b200.utils.env import TUNED

    print("# more bytes in flight per channel for large messages (NCCL's proxy pipeline is the limit, not the link):", file=out)
    print("export " + " ".join(f"{k}={v}" for k, v in TUNED.items()), file=out)
    print("# expect in the log (NCCL_DEBUG=INFO): 'NET/Plugin: Loaded net plugin BNet (v8)' and 'Using network BNet'", file=out)
    return 1 if problems else 0


if __name__ == "__main__":
    sys.exit(run())

#!/usr/bin/env python
"""Which CUDA calls block while a long-running kernel occupies the device?

A transport that serves NCCL must never issue such a call on the data path: the NCCL kernel
that is running is waiting for the transport, so a call that waits for the device to drain is a
dead-lock.  This probe starts a ~1.5 s spinning kernel on GPU 0 and times each candidate call
issued right after it (fresh spin per call).  "BLOCKED" = the call returned only when the spin
was over.  Needs 1 GPU (peer/IPC imports come from a helper process on the same GPU).

  python tools/blocking_calls_probe.py [--out profiles/blocking_calls.txt]
"""
import argparse
import array
import os
import socket
import subprocess
import sys
import time
import warnings

warnings.filterwarnings("ignore")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SPIN_S = 1.5


def child(sock_path):
    """Exporter: one cudaMalloc buffer (legacy IPC handle) + one cuMemCreate buffer (POSIX fd)."""
    from cuda import cuda, cudart

    cudart.cudaSetDevice(0)
    cudart.cudaFree(0)
    err, p = cudart.cudaMalloc(64 << 20)
    err, ipc = cudart.cudaIpcGetMemHandle(p)
    prop = cuda.CUmemAllocationProp()
    prop.type = cuda.CUmemAllocationType.CU_MEM_ALLOCATION_TYPE_PINNED
    prop.location.type = cuda.CUmemLocationType.CU_MEM_LOCATION_TYPE_DEVICE
    prop.location.id = 0
    prop.requestedHandleTypes = cuda.CUmemAllocationHandleType.CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR
    err, gran = cuda.cuMemGetAllocationGranularity(prop, cuda.CUmemAllocationGranularity_flags.CU_MEM_ALLOC_GRANULARITY_RECOMMENDED)
    size = max(gran, 64 << 20) // gran * gran
    fds = []
    for _ in range(3):
        err, h = cuda.cuMemCreate(size, prop, 0)
        err, fd = cuda.cuMemExportToShareableHandle(h, cuda.CUmemAllocationHandleType.CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0)
        fds.append(int(fd))
    s = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    s.connect(sock_path)
    payload = bytes(ipc.reserved) + size.to_bytes(8, "little")
    socket.send_fds(s, [payload], fds)
    s.recv(1)   # parent says we can go
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--child", default="")
    a = ap.parse_args()
    if a.child:
        return child(a.child)

    import torch
    from cuda import cuda, cudart

    torch.cuda.set_device(0)
    torch.zeros(1, device="cuda")
    clock_khz = torch.cuda.get_device_properties(0).clock_rate if hasattr(torch.cuda.get_device_properties(0), "clock_rate") else 1965000
    cycles = int(SPIN_S * 1.9e9)
    spin_stream = torch.cuda.Stream()
    side = torch.cuda.Stream()

    # helper process with exportable allocations
    path = f"/tmp/bnet-probe-{os.getpid()}.sock"
    srv = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
    srv.bind(path)
    srv.listen(1)
    proc = subprocess.Popen([sys.executable, os.path.abspath(__file__), "--child", path])
    conn, _ = srv.accept()
    msg, fds, _, _ = socket.recv_fds(conn, 4096, 8)
    ipc_bytes, size = msg[:64], int.from_bytes(msg[64:72], "little")

    results = []

    def probe(name, fn):
        torch.cuda.synchronize()
        with torch.cuda.stream(spin_stream):
            torch.cuda._sleep(cycles)
        t0 = time.perf_counter()
        try:
            extra = fn()
        except Exception as e:   # noqa: BLE001
            extra = f"EXC {type(e).__name__}: {e}"
        dt = time.perf_counter() - t0
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        verdict = "BLOCKED" if dt > 0.6 * total and total > 0.5 else "ok"
        results.append((name, dt * 1e3, total * 1e3, verdict, extra))
        print(f"{name:46s} {dt * 1e3:9.2f} ms (spin ended at {total * 1e3:7.1f} ms)  {verdict}  {extra if extra else ''}", flush=True)

    def kernel_other_stream():
        with torch.cuda.stream(side):
            x = torch.ones(1 << 20, device="cuda")
            x.add_(1)
            ev = torch.cuda.Event()
            ev.record()
        t0 = time.perf_counter()
        while not ev.query() and time.perf_counter() - t0 < 3:
            pass
        return f"side-stream kernel finished after {(time.perf_counter() - t0) * 1e3:.1f} ms"

    def memcpy_other_stream():
        h = torch.empty(1 << 20, dtype=torch.uint8).pin_memory()
        with torch.cuda.stream(side):
            d = h.to("cuda", non_blocking=True)
            side.synchronize()
        return ""

    probe("kernel launch + completion on another stream", kernel_other_stream)
    probe("cudaHostAlloc + cudaMemcpyAsync(other stream)+sync", memcpy_other_stream)
    probe("cudaStreamCreateWithPriority", lambda: cudart.cudaStreamCreateWithPriority(cudart.cudaStreamNonBlocking, -1)[0])
    probe("cudaMalloc(64 MiB)", lambda: cudart.cudaMalloc(64 << 20)[0])
    probe("cudaHostAlloc(1 MiB, mapped)", lambda: cudart.cudaHostAlloc(1 << 20, cudart.cudaHostAllocMapped)[0])
    buf = bytearray(1 << 20)
    addr = (array.array("B", buf)).buffer_info()[0]

    POSIX = cuda.CUmemAllocationHandleType.CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR
    state = {}

    def imp(i):
        err, h = cuda.cuMemImportFromShareableHandle(fds[i], POSIX)
        state[f"h{i}"] = h
        return str(err)

    def reserve(i):
        err, va = cuda.cuMemAddressReserve(size, 0, 0, 0)
        state[f"va{i}"] = va
        return str(err)

    def do_map(i):
        return str(cuda.cuMemMap(state[f"va{i}"], size, 0, state[f"h{i}"], 0)[0])

    def set_access(i):
        acc = cuda.CUmemAccessDesc()
        acc.location.type = cuda.CUmemLocationType.CU_MEM_LOCATION_TYPE_DEVICE
        acc.location.id = 0
        acc.flags = cuda.CUmemAccess_flags.CU_MEM_ACCESS_FLAGS_PROT_READWRITE
        return str(cuda.cuMemSetAccess(state[f"va{i}"], size, [acc], 1)[0])

    probe("cuMemImportFromShareableHandle (peer fd)", lambda: imp(0))
    probe("cuMemAddressReserve", lambda: reserve(0))
    probe("cuMemMap (imported handle)", lambda: do_map(0))
    probe("cuMemSetAccess (imported mapping)", lambda: set_access(0))

    def whole_import():
        return " ".join([imp(1), reserve(1), do_map(1), set_access(1)])

    probe("import+reserve+map+setaccess in one go", whole_import)

    def ipc_open():
        hdl = cudart.cudaIpcMemHandle_t()
        hdl.reserved = ipc_bytes
        err, p = cudart.cudaIpcOpenMemHandle(hdl, cudart.cudaIpcMemLazyEnablePeerAccess)
        state["ipc"] = p
        return str(err)

    probe("cudaIpcOpenMemHandle (peer cudaMalloc)", ipc_open)
    probe("cuMemUnmap", lambda: str(cuda.cuMemUnmap(state["va0"], size)[0]))
    probe("cuMemRelease", lambda: str(cuda.cuMemRelease(state["h0"])[0]))
    probe("cuMemAddressFree", lambda: str(cuda.cuMemAddressFree(state["va0"], size)[0]))
    probe("cudaIpcCloseMemHandle", lambda: str(cudart.cudaIpcCloseMemHandle(state["ipc"])[0]) if "ipc" in state else "n/a")
    probe("cudaHostRegister(1 MiB)", lambda: str(cudart.cudaHostRegister(addr, 1 << 20, cudart.cudaHostRegisterMapped)[0]))

    # our own executor: cluster-kernel launch (one-shot) while the device is busy
    def exec_copy():
        from bagua_net_b200.ops import P2PExecutor

        ex = state.setdefault("ex", P2PExecutor(0))
        a_ = state.setdefault("a", torch.ones(1 << 20, device="cuda"))
        b_ = state.setdefault("b", torch.zeros(1 << 20, device="cuda"))
        t0 = time.perf_counter()
        ex.wait(ex.submit("copy", a_, b_, sync=False), timeout=5)
        return f"bnet cluster kernel completed after {(time.perf_counter() - t0) * 1e3:.1f} ms"

    torch.cuda.synchronize()
    exec_copy()
    probe("bnet executor: cluster kernel launch + completion", exec_copy)

    # ---- second question: while ANOTHER thread sits in a device-synchronising call (cudaFree as issued
    # by torch's emptyCache after a cuDNN benchmark, ...), can this thread still launch / map / copy?
    import threading

    warm = torch.ones(1 << 20, device="cuda")
    with torch.cuda.stream(side):
        warm.add_(1)
    torch.cuda.synchronize()

    def concurrent(xname, xfn, yname, yfn):
        torch.cuda.synchronize()
        with torch.cuda.stream(spin_stream):
            torch.cuda._sleep(cycles)
        t0 = time.perf_counter()
        xdone = {}

        def run_x():
            xfn()
            xdone["t"] = time.perf_counter() - t0

        th = threading.Thread(target=run_x)
        th.start()
        time.sleep(0.05)
        ty0 = time.perf_counter()
        try:
            extra = yfn()
        except Exception as e:   # noqa: BLE001
            extra = f"EXC {e}"
        ty = time.perf_counter() - ty0
        th.join()
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        verdict = "BLOCKED" if ty > 0.5 * total else "ok"
        line = (f"[{xname} in thread A: returned after {xdone.get('t', -1) * 1e3:7.1f} ms]  {yname}: {ty * 1e3:8.2f} ms  {verdict}  {extra or ''}")
        results.append((f"A={xname} | B={yname}", ty * 1e3, total * 1e3, verdict, extra))
        print(line, flush=True)

    def y_launch():
        with torch.cuda.stream(side):
            warm.add_(1)
            ev = torch.cuda.Event()
            ev.record()
        t0 = time.perf_counter()
        while not ev.query() and time.perf_counter() - t0 < 3:
            pass
        return f"kernel completed {(time.perf_counter() - t0) * 1e3:.1f} ms after launch returned"

    def y_exec():
        return exec_copy()

    def y_import():
        return " ".join([imp(2), reserve(2), do_map(2), set_access(2)])

    def y_memcpy():
        h = state.setdefault("pinned", torch.empty(1 << 20, dtype=torch.uint8).pin_memory())
        with torch.cuda.stream(side):
            h.to("cuda", non_blocking=True)
            side.synchronize()
        return ""

    def x_cudafree():
        err, p = cudart.cudaMalloc(256 << 20)
        state["tofree"] = p

    xs = {
        "cudaFree": lambda: cudart.cudaFree(state.pop("tofree")),
        "cudaDeviceSynchronize": lambda: cudart.cudaDeviceSynchronize(),
        "torch.cuda.empty_cache": lambda: torch.cuda.empty_cache(),
    }
    for xname, xfn in xs.items():
        for yname, yfn in (("kernel launch (loaded)", y_launch), ("bnet cluster kernel", y_exec), ("cudaMemcpyAsync+sync", y_memcpy)):
            if xname == "cudaFree":
                x_cudafree()
            if xname == "torch.cuda.empty_cache":
                _ = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
                del _
            concurrent(xname, xfn, yname, yfn)
    x_cudafree()
    concurrent("cudaFree", xs["cudaFree"], "cuMem import+map+setaccess", y_import)

    conn.send(b"x")
    proc.wait(timeout=20)
    os.unlink(path)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(f"# CUDA calls issued while a {SPIN_S}s kernel runs on the same device ({torch.cuda.get_device_name()}, CUDA {torch.version.cuda})\n")
            for name, dt, total, verdict, extra in results:
                f.write(f"{name:52s} {dt:9.2f} ms  {verdict:8s} {extra}\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())

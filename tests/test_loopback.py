"""ABI + transport tests over loopback, two processes — BASELINE.json config #1
("ncclNet_v4 loopback isend/irecv correctness, 2 ranks on CPU sockets") widened to every
exported ABI version, both TCP backends, the shared-memory (NVL) transport, 8 requests
in flight, sizes around the chunking boundaries, receive buffers larger than the message.
The reference has no such test (SURVEY.md §4: BASIC backend tests: none)."""
import os

import pytest

from conftest import run_pair

SIZES = "0,1,8,4096,524288,1048575,1048577,3145729"


def _check(outs, transport=None):
    for rc, res, err in outs:
        assert res is not None, err
        assert rc == 0 and res["ok"], (res, err[-2000:])
        assert res["name"] == "BNet"
        if transport:
            assert res["transport"] == transport, res
    return outs


@pytest.mark.parametrize("abi", [3, 4, 6, 8])
def test_abi_versions_tcp_basic(abi):
    _check(run_pair(["--abi", str(abi), "--sizes", SIZES, "--inflight", "8", "--rounds", "1"],
                    env={"BNET_NVL": "0"}), "tcp-threads")


def test_abi_v10_table():
    # exported only by the -bnetx variant; layout checked through the same driver
    import ctypes
    import os

    import bagua_net_b200
    from bagua_net_b200.utils.abi import NetPlugin

    p = NetPlugin(10, "libnccl-net-bnetx.so")
    p.init()
    props = p.get_properties(0)
    assert props["maxRecvs"] == 1 and props["vProps"]["ndevs"] == 1 and props["maxP2pBytes"] > 1 << 30
    assert os.path.exists(bagua_net_b200.lib_path("libnccl-net-bnet.so"))
    lib = ctypes.CDLL(bagua_net_b200.lib_path())
    for v in (3, 4, 5, 6, 7, 8):
        assert hasattr(lib, f"ncclNetPlugin_v{v}")
    if "BNET_LIB_DIR" not in os.environ:              # (the sanitizer builds put every table into one library)
        assert not hasattr(lib, "ncclNetPlugin_v10")  # default build stays on well-known layouts


def test_v10_profiler_callback_brackets_every_request():
    """ncclNet v10: init() receives NCCL's profiler callback, isend/irecv a parent event handle; the plugin opens one
    event per request under it and closes it when test() reports completion (include/bnet/bnet_profiler.h)."""
    import ctypes as C

    import numpy as np

    from bagua_net_b200.utils.abi import BNET_PROFILER_PLUGIN_ID, PROFILER_CB, NetPlugin, ProfilerEventDescr

    events = []
    handles = iter(range(0x1000, 0x2000))

    def cb(ehandle, typ, phandle, plugin_id, ext):
        d = C.cast(ext, C.POINTER(ProfilerEventDescr)).contents
        if typ == 0:
            ehandle[0] = next(handles)
        events.append((typ, ehandle[0], phandle, plugin_id, d.type, d.path, d.length, d.comm_id))
        return 0

    prof = PROFILER_CB(cb)
    p = NetPlugin(10, "libnccl-net-bnetx.so")
    p.init(profiler=prof)
    h, l = p.listen(0)
    s = p.connect(h)
    r = p.accept(l)
    src, dst = np.arange(70000, dtype=np.uint8), np.zeros(70000, dtype=np.uint8)
    rq = p.irecv(r, dst.ctypes.data, 70000, phandle=0xAAAA)
    sq = p.isend(s, src.ctypes.data, 70000, phandle=0xBBBB)
    q2 = p.isend(s, src.ctypes.data, 16)                      # no parent handle: no profiler event
    r2 = p.irecv(r, dst.ctypes.data, 16)
    assert p.wait(sq) == 70000 and p.wait(rq) == 70000 and p.wait(q2) == 16 and p.wait(r2) == 16
    p.close_send(s), p.close_recv(r), p.close_listen(l)
    starts = [e for e in events if e[0] == 0]
    stops = [e for e in events if e[0] == 1]
    assert len(starts) == 2 and len(stops) == 2
    assert {e[2] for e in starts} == {0xAAAA, 0xBBBB} and all(e[3] == BNET_PROFILER_PLUGIN_ID for e in events)
    assert {e[1] for e in starts} == {e[1] for e in stops}               # every event that was opened is closed
    assert {e[4] for e in starts} == {0, 1}                                # one isend, one irecv
    assert all(e[6] == 70000 for e in stops) and all(e[5] in (0, 1, 2, 3) for e in stops)


@pytest.mark.parametrize("nstreams", [1, 2, 8])
@pytest.mark.parametrize("impl", ["BASIC", "TOKIO"])
def test_tcp_backends_and_nstreams(impl, nstreams):
    env = {"BNET_NVL": "0", "BAGUA_NET_IMPLEMENT": impl, "BAGUA_NET_NSTREAMS": str(nstreams),
           "BAGUA_NET_MIN_CHUNKSIZE": "65536"}
    _check(run_pair(["--sizes", SIZES, "--inflight", "8", "--rounds", "2"], env=env),
           "tcp-threads" if impl == "BASIC" else "tcp-async")


def test_sender_params_win_over_receiver_params():
    # The reference silently corrupts data when both ends disagree on NSTREAMS/MIN_CHUNKSIZE
    # (SURVEY.md §2.2 protocol invariant).  Here the preamble carries the sender's values.
    import json
    import os
    import subprocess
    import sys
    import tempfile

    from conftest import ROOT

    worker = os.path.join(ROOT, "tests", "loopback_worker.py")
    base = dict(os.environ, PYTHONPATH=ROOT, BNET_NVL="0")
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.Popen([sys.executable, worker, "0", d, "--sizes", "1048577,3145729"],
                             env=dict(base, BAGUA_NET_NSTREAMS="2", BAGUA_NET_MIN_CHUNKSIZE="1048576"),
                             stdout=subprocess.PIPE, text=True)
        s = subprocess.Popen([sys.executable, worker, "1", d, "--sizes", "1048577,3145729"],
                             env=dict(base, BAGUA_NET_NSTREAMS="5", BAGUA_NET_MIN_CHUNKSIZE="4096",
                                      BAGUA_NET_IMPLEMENT="TOKIO"),
                             stdout=subprocess.PIPE, text=True)
        ro, so = r.communicate(timeout=120)[0], s.communicate(timeout=120)[0]
    rres, sres = json.loads(ro.splitlines()[-1]), json.loads(so.splitlines()[-1])
    assert rres["ok"] and sres["ok"], (rres, sres)
    assert rres["transport"] == "tcp-async"        # receiver followed the sender's backend too


def test_wire_compat_mode():
    # bare reference framing: 8-byte BE stream id preamble, sockaddr-only handle
    _check(run_pair(["--abi", "4", "--sizes", "0,8,1048577", "--inflight", "4", "--rounds", "1"],
                    env={"BNET_WIRE_COMPAT": "1", "BNET_NVL": "0"}), "tcp-threads")


@pytest.mark.parametrize("impl", ["BASIC", "TOKIO"])
@pytest.mark.parametrize("ours", ["receiver", "sender"])
@pytest.mark.parametrize("streams", [(2, None), (5, 4096)])
def test_interoperates_with_a_peer_that_speaks_the_reference_format(impl, ours, streams):
    """The other end is tests/ref_wire_peer.py: the reference's wire format re-implemented from its specification with plain
    Python sockets (handle = bare sockaddr, 8-byte stream ids, u64 / u32 length framing, the reference's chunking and
    stream cursor).  The plugin is driven through the reference's ABI (ncclNet v4) with BNET_WIRE_COMPAT=1."""
    import json
    import subprocess
    import sys
    import tempfile
    import threading
    import time

    from conftest import ROOT
    from loopback_worker import pattern
    from ref_wire_peer import RefReceiver, RefSender

    sizes, inflight, rounds = [0, 8, 65536, 1048577, 3145729], 4, 2
    worker = os.path.join(ROOT, "tests", "loopback_worker.py")
    env = dict(os.environ, PYTHONPATH=ROOT, BNET_NVL="0", BNET_WIRE_COMPAT="1", BAGUA_NET_IMPLEMENT=impl)
    env.pop("BAGUA_NET_NSTREAMS", None)
    env.pop("BAGUA_NET_MIN_CHUNKSIZE", None)
    nstreams, min_chunk = streams          # (the reference's defaults / five streams and chunks from 4 KiB: both ends set alike)
    if min_chunk is not None:
        env.update(BAGUA_NET_NSTREAMS=str(nstreams), BAGUA_NET_MIN_CHUNKSIZE=str(min_chunk))
    messages = [bytes(pattern(size, 1000 * rnd + 7 * j + size % 97)[:size])
                for rnd in range(rounds) for size in sizes for j in range(inflight)]
    args = ["--abi", "4", "--sizes", ",".join(map(str, sizes)), "--inflight", str(inflight), "--rounds", str(rounds)]
    with tempfile.TemporaryDirectory() as d:
        hfile = os.path.join(d, "handle.bin")
        if ours == "receiver":
            proc = subprocess.Popen([sys.executable, worker, "0", d] + args, env=env, stdout=subprocess.PIPE, text=True)
            t0 = time.time()
            while not os.path.exists(hfile):
                assert time.time() - t0 < 60 and proc.poll() is None, "the plugin's listener did not come up"
                time.sleep(0.01)
            handle = open(hfile, "rb").read()
            assert handle[28:32] == b"\0\0\0\0"            # (no magic: a bare sockaddr, as the reference's handle)
            peer = RefSender(handle, impl, nstreams, min_chunk)
            err = []

            def feed():
                try:
                    for m in messages:
                        peer.send(m)
                except Exception as ex:   # noqa: BLE001
                    err.append(ex)

            th = threading.Thread(target=feed, daemon=True)
            th.start()
            out = proc.communicate(timeout=120)[0]
            th.join(timeout=30)
            peer.close()
            assert not err, err
        else:
            peer = RefReceiver(impl, nstreams, min_chunk)
            with open(hfile + ".tmp", "wb") as f:
                f.write(peer.handle)
            os.rename(hfile + ".tmp", hfile)
            proc = subprocess.Popen([sys.executable, worker, "1", d] + args, env=env, stdout=subprocess.PIPE, text=True)
            peer.accept()
            for i, m in enumerate(messages):
                got = peer.recv()
                assert got == m, f"message {i}: {len(got)} bytes, expected {len(m)}"
            out = proc.communicate(timeout=120)[0]
            peer.close()
    res = json.loads(out.splitlines()[-1])
    assert res["ok"] and res["messages"] == len(messages), res
    assert res["transport"] == ("tcp-threads" if impl == "BASIC" else "tcp-async")


def test_nvl_shared_memory_host_buffers():
    _check(run_pair(["--sizes", SIZES + ",9437184", "--inflight", "8", "--rounds", "2"],
                    env={"BNET_NVL": "1", "BNET_SHM_RING_BYTES": "1048576"}), "nvl")


def test_nvl_large_host_messages_are_pulled_with_one_copy():
    # same-host, host buffers, >= 512 KiB: the receiver reads the payload straight out of the sender's buffer
    # (process_vm_readv, probed at accept); smaller messages and BNET_CMA=0 keep using the ring
    args = ["--sizes", "0,8,524287,524288,1048577,9437184", "--inflight", "8", "--rounds", "2"]
    on = _check(run_pair(args, env={"BNET_NVL": "1"}), "nvl")
    assert on[1][1]["cma_messages"] == 8 * 2 * 3, on[1][1]
    off = _check(run_pair(args, env={"BNET_NVL": "1", "BNET_CMA": "0"}), "nvl")
    assert off[1][1]["cma_messages"] == 0, off[1][1]


def test_nvl_direct_path_with_emulated_device_memory():
    # regMr(NCCL_PTR_CUDA) export/import, FIFO matching and per-chunk completion words,
    # with "device memory" emulated by shm segments (BNET_FAKE_CUDA=1)
    outs = _check(run_pair(["--mem", "fakecuda", "--sizes", "0,1,8,4096,1048577,3145729", "--inflight", "8",
                            "--rounds", "2"], env={"BNET_NVL": "1", "BNET_FAKE_CUDA": "1"}), "nvl")
    assert outs[0][1]["messages"] == 96


@pytest.mark.parametrize("name,env,extra,transport", [
    ("tcp-basic", {"BNET_NVL": "0"}, [], "tcp-threads"),
    ("tcp-async", {"BNET_NVL": "0", "BAGUA_NET_IMPLEMENT": "TOKIO"}, [], "tcp-async"),
    ("nvl-host", {"BNET_NVL": "1"}, [], "nvl"),
    ("nvl-device", {"BNET_NVL": "1", "BNET_FAKE_CUDA": "1"}, ["--mem", "fakecuda"], "nvl")])
@pytest.mark.parametrize("abi", [6, 8])
def test_grouped_receives(name, env, extra, transport, abi):
    """ncclNet v5+ `irecv(n > 1)` (`maxRecvs`, BNET_MAX_RECVS): n buffers under one request, filled in order by the sender's
    next n isends (NCCL gives every entry of a group the same tag), `test` reports n sizes; a last, shorter group included."""
    outs = _check(run_pair(["--abi", str(abi), "--sizes", "0,1,4096,1048577", "--inflight", "7", "--rounds", "2", "--group", "3"] + extra,
                           env=dict(env, BNET_MAX_RECVS="8")), transport)
    assert outs[0][1]["grouped"] == 3 * 4 * 2 and outs[0][1]["messages"] == 7 * 4 * 2, outs[0][1]


def test_max_recvs_property_follows_the_knob():
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("from bagua_net_b200.utils.abi import NetPlugin\n"
            "p = NetPlugin(8); p.init(); print('maxRecvs', p.get_properties(0)['maxRecvs'])")
    for knob, want in ((None, 1), ("8", 8), ("99", 8)):
        env = {k: v for k, v in os.environ.items() if k != "BNET_MAX_RECVS"}
        env["PYTHONPATH"] = root + os.pathsep + env.get("PYTHONPATH", "")
        if knob:
            env["BNET_MAX_RECVS"] = knob
        out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
        assert out.returncode == 0 and f"maxRecvs {want}" in out.stdout, (knob, out.stdout, out.stderr[-1500:])


def test_nvl_pinned_host_source_goes_direct_when_enabled():
    # NCCL keeps its LL send buffers in pinned host memory; with BNET_HOST_SRC_DIRECT=1 the copy kernel reads them
    # through their device alias and stores into the peer's device buffer (emulated here), no ring, no staging
    args = ["--mem", "fakecuda", "--send-mem", "host", "--sizes", "0,1,8,4096,1048577", "--inflight", "8", "--rounds", "2"]
    on = _check(run_pair(args, env={"BNET_NVL": "1", "BNET_FAKE_CUDA": "1", "BNET_HOST_SRC_DIRECT": "1"}), "nvl")
    assert on[1][1]["kernel_chunks"] > 0, on[1][1]
    off = _check(run_pair(args, env={"BNET_NVL": "1", "BNET_FAKE_CUDA": "1"}), "nvl")
    assert off[1][1]["kernel_chunks"] == 0, off[1][1]


@pytest.mark.parametrize("direct", ["0", "1"])
def test_nvl_ring_and_direct_messages_interleaved_on_one_connection(direct):
    # NCCL alternates protocols on a connection over time (LL: pinned host source, Simple: device source); ring-path
    # and direct-path messages must stay FIFO with 8 requests in flight
    _check(run_pair(["--mem", "fakecuda", "--mix", "--sizes", "0,8,4096,70000,1048577", "--inflight", "8", "--rounds", "3"],
                    env={"BNET_NVL": "1", "BNET_FAKE_CUDA": "1", "BNET_HOST_SRC_DIRECT": direct}), "nvl")


def test_cuda_pointers_over_tcp_are_staged():
    _check(run_pair(["--mem", "fakecuda", "--sizes", "1,4096,1048577,3145729", "--inflight", "4", "--rounds", "1"],
                    env={"BNET_NVL": "0", "BNET_FAKE_CUDA": "1"}), "tcp-threads")
    _check(run_pair(["--mem", "fakecuda", "--sizes", "1,4096,1048577", "--inflight", "4", "--rounds", "1"],
                    env={"BNET_NVL": "0", "BNET_FAKE_CUDA": "1", "BAGUA_NET_IMPLEMENT": "TOKIO"}), "tcp-async")


@pytest.mark.parametrize("env", [{"BNET_NVL": "0"}, {"BNET_NVL": "0", "BAGUA_NET_IMPLEMENT": "TOKIO"},
                                 {"BNET_NVL": "1"}])
def test_peer_death_is_an_error_not_a_hang(env):
    # fault injection the reference lacks (SURVEY.md §5.3: data-stream errors hang there)
    outs = run_pair(["--sizes", "4194304", "--inflight", "8", "--rounds", "4", "--die-after", "9"],
                    env=dict(env, BNET_SHM_RING_BYTES="262144"), timeout=60)
    rc, res, err = outs[0]          # receiver
    assert res is not None and not res["ok"], (res, err[-1000:])
    assert res["code"] in (2, 6), res      # ncclSystemError / ncclRemoteError


def test_injected_stream_failure_surfaces_in_test():
    outs = run_pair(["--sizes", "2097152", "--inflight", "4", "--rounds", "3"],
                    env={"BNET_NVL": "0", "BNET_FAULT_INJECT": "send_drop_after=3", "BAGUA_NET_MIN_CHUNKSIZE": "65536"},
                    timeout=60)
    assert any(res is not None and not res["ok"] for _, res, _ in outs)


# ---- N ranks, two different peers per rank, several connections per peer (what NCCL's rings look like)
@pytest.mark.parametrize("world,env,args,transport", [
    (4, {"BNET_NVL": "0"}, ["--channels", "2"], "tcp-threads"),
    (3, {"BNET_NVL": "0", "BAGUA_NET_IMPLEMENT": "TOKIO", "BAGUA_NET_NSTREAMS": "3"}, ["--channels", "2"], "tcp-async"),
    (4, {}, ["--channels", "2", "--mem", "host"], "nvl"),
    (8, {"BNET_FAKE_CUDA": "1"}, ["--channels", "4", "--mem", "fakecuda", "--iters", "2"], "nvl"),
    (3, {"BNET_FAKE_CUDA": "1"}, ["--channels", "1", "--slices", "1", "--mem", "fakecuda"], "nvl"),
])
def test_ring_allreduce_over_the_plugin(world, env, args, transport):
    from conftest import run_ring

    outs = run_ring(world, args, env=env)
    for rc, res, err in outs:
        assert rc == 0 and res and res["ok"], err[-2000:]
        assert res["transports"] == [transport]
        assert res["allreduces"] > 0


def test_listener_survives_garbage_connections():
    """Port scanners / half-open connections / random bytes on the listening socket must neither produce a comm
    nor block the next genuine connect (the reference would read them as stream ids: nthread_…:440-447)."""
    import subprocess
    import sys

    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "scripts", "garbage_connections.py")
    r = subprocess.run([sys.executable, script], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "ok after garbage" in r.stdout, r.stdout[-1500:] + r.stderr[-1500:]


@pytest.mark.skipif(not os.path.exists("/proc/net/if_inet6") or " lo" not in open("/proc/net/if_inet6").read(),
                    reason="no IPv6 loopback address")
@pytest.mark.parametrize("abi", [4, 8])
def test_ipv6_listener_handle_is_not_truncated(abi):
    # the reference copies a 16-byte `struct sockaddr` into the handle, which cuts a sockaddr_in6 (lib.rs:157-158);
    # ours keeps all 28 bytes even in the 64-byte v4 handle
    _check(run_pair(["--abi", str(abi), "--sizes", "0,8,1048577", "--inflight", "4", "--rounds", "1"],
                    env={"BNET_NVL": "0", "NCCL_SOCKET_IFNAME": "lo", "NCCL_SOCKET_FAMILY": "10"}), "tcp-threads")


def test_async_backend_lends_large_chunks_to_other_loops():
    # >= 3 chunks of >= 512 KiB each: the epoll backend hands the chunks to helper loops of its pool for the
    # duration of the chunk (tcp_async.cc); message-serial order and byte placement must not change
    _check(run_pair(["--sizes", "1572864,6291459,16777216,4096", "--inflight", "4", "--rounds", "2"],
                    env={"BNET_NVL": "0", "BAGUA_NET_IMPLEMENT": "TOKIO", "BAGUA_NET_NSTREAMS": "4"}), "tcp-async")
    _check(run_pair(["--sizes", "8388608", "--inflight", "8", "--rounds", "2"],
                    env={"BNET_NVL": "0", "BAGUA_NET_IMPLEMENT": "TOKIO", "BAGUA_NET_NSTREAMS": "8",
                         "BAGUA_NET_TOKIO_WORKER_THREADS": "3"}), "tcp-async")


def test_async_backend_peer_death_while_chunks_are_lent():
    outs = run_pair(["--sizes", "16777216", "--inflight", "8", "--rounds", "4", "--die-after", "11", "--expect-error"],
                    env={"BNET_NVL": "0", "BAGUA_NET_IMPLEMENT": "TOKIO", "BAGUA_NET_NSTREAMS": "4"}, timeout=120)
    rc, res, err = outs[0]          # the receiver must see an error, not hang
    assert rc == 0 and res is not None and not res["ok"], (res, err[-2000:])


def _random_sizes(seed, n):
    import random

    rnd = random.Random(seed)
    out = []
    for _ in range(n):
        r = rnd.random()
        out.append(rnd.randint(0, 64) if r < 0.2 else rnd.randint(65, 70000) if r < 0.6 else
                   rnd.randint(70001, 1200000) if r < 0.9 else rnd.randint(1200001, 5000000))
    return ",".join(map(str, out))


@pytest.mark.parametrize("name,env,extra", [
    ("tcp-threads", {"BNET_NVL": "0", "BAGUA_NET_NSTREAMS": "3"}, []),
    ("tcp-async", {"BNET_NVL": "0", "BAGUA_NET_IMPLEMENT": "TOKIO", "BAGUA_NET_NSTREAMS": "5", "BAGUA_NET_MIN_CHUNKSIZE": "100000"}, []),
    ("nvl", {"BNET_NVL": "1", "BNET_SHM_RING_BYTES": "131072"}, []),
    ("nvl", {"BNET_NVL": "1", "BNET_FAKE_CUDA": "1", "BNET_HOST_SRC_DIRECT": "1"}, ["--mem", "fakecuda", "--mix"]),
], ids=["basic", "epoll", "shm-ring+cma", "emulated-device-mix"])
def test_random_message_sizes(name, env, extra):
    # 100 messages of random sizes (0 B .. 5 MB), 8 in flight, every byte checked
    _check(run_pair(["--sizes", _random_sizes(7, 100), "--inflight", "8", "--rounds", "1"] + extra, env=env, timeout=300), name)


@pytest.mark.parametrize("env", [{"BNET_NVL": "0"}, {"BNET_NVL": "0", "BAGUA_NET_IMPLEMENT": "TOKIO"}, {"BNET_NVL": "1"}],
                         ids=["basic", "epoll", "nvl"])
def test_connection_churn_leaks_nothing(env):
    # 60 listen/connect/accept/regMr/transfer/close cycles in one process: fds, threads and /dev/shm stay flat
    import subprocess
    import sys

    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "scripts", "fd_leak.py")
    r = subprocess.run([sys.executable, script, "60"], capture_output=True, text=True, timeout=300, env=dict(os.environ, **env))
    assert r.returncode == 0 and "no leak" in r.stdout, r.stdout[-1500:] + r.stderr[-1500:]


def test_per_gpu_virtual_devices():
    """Device model of SURVEY section 5.8: one virtual net device per GPU (pciPath = the GPU's, so NCCL places it next to
    that GPU and enables GPUDirect on its own), NIC devices after them.  Checked here with the emulated CUDA side."""
    import json
    import os
    import subprocess
    import sys

    code = ("import json\n"
            "from bagua_net_b200.utils.abi import NetPlugin\n"
            "p = NetPlugin(8); p.init(); n = p.devices()\n"
            "print(json.dumps([p.get_properties(i) for i in range(n)]))\n")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNET_FAKE_CUDA="1", BNET_GPU_DEVICES="1", BNET_NVL="1", PYTHONPATH=root)
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    props = json.loads(out.stdout.splitlines()[-1])
    assert len(props) >= 2
    g = props[0]
    assert g["name"] == "bnet-gpu0" and g["ptrSupport"] == 3 and g["speed"] == 3600000 and g["maxRecvs"] == 1
    assert not g["pciPath"]        # a virtual NVLink "NIC" has no PCI leaf of its own (never the GPU's: see engine.cc)
    assert all(not p["name"].startswith("bnet-gpu") for p in props[1:])           # the NIC devices follow
    assert len({p["guid"] for p in props}) == len(props)
    # and the default without a GPU: NIC devices only, like the reference (nthread_…:241-257)
    env2 = dict(os.environ, BNET_GPU_DEVICES="1", PYTHONPATH=root)
    env2.pop("BNET_FAKE_CUDA", None)
    out = subprocess.run([sys.executable, "-c", code], env=env2, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr[-2000:]
    assert not any(p["name"].startswith("bnet-gpu") for p in json.loads(out.stdout.splitlines()[-1]))


def _run_tring(world, count, dtype, piece, inflight, timeout=180, extra_env=None):
    import json
    import subprocess
    import sys
    import tempfile

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNET_FAKE_CUDA="1", BNET_NVL="1", PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    env.update(extra_env or {})
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, os.path.join(root, "tests", "tring_worker.py"), str(r), str(world), d, str(count),
                                   dtype, str(piece), str(inflight)], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
                 for r in range(world)]
        outs = []
        for p in procs:
            try:
                o, e = p.communicate(timeout=timeout)
            except subprocess.TimeoutExpired:
                for q in procs:
                    q.kill()
                raise
            assert p.returncode == 0, e[-3000:]
            outs.append(json.loads([ln for ln in o.splitlines() if ln.startswith("{")][-1]))
    return outs


@pytest.mark.parametrize("world,count,dtype,piece,inflight", [
    (2, 1 << 16, "f32", 16384, 4), (3, 100003, "f32", 8192, 8), (4, 1 << 18, "bf16", 65536, 16), (5, 7, "f32", 4096, 2),
    (8, 300000, "bf16", 32768, 16)])
def test_transport_ring_allreduce_with_fused_isend_reduce(world, count, dtype, piece, inflight):
    """The all-reduce that rides the transport: reduce-scatter hops are isend_op(OP_RED_ADD_*) — the receiver's registered
    buffer is accumulated into by the sender's kernel (here: its CPU emulation) — all-gather hops plain isends; pieces
    pipeline around the ring with many requests in flight.  Bit-exact against the closed-form sum."""
    outs = _run_tring(world, count, dtype, piece, inflight)
    assert all(o["ok"] for o in outs), outs
    assert all(o["transport"] == "nvl" for o in outs)
    assert all(o["stats"]["messages"] >= 2 * (world - 1) for o in outs)


@pytest.mark.parametrize("world,count,wire,fused,piece,inflight", [
    (2, 1 << 16, "bf16", 1, 16384, 4), (3, 100003, "e4m3", 1, 8192, 8), (4, 1 << 18, "e4m3", 0, 65536, 16),
    (5, 777, "bf16", 0, 4096, 2), (8, 300000, "e4m3", 1, 32768, 16), (4, 50000, "e5m2", 1, 4096, 8)])
def test_transport_ring_compressed_allreduce(world, count, wire, fused, piece, inflight):
    """fp32 all-reduce with a narrower format on the wire (K5: the cast fused into the transport).  Fused mode: every
    reduce-scatter hop is isend_op(OP_CAST_F32_TO_<wire>) into the next rank's wire mirror, the receiver accumulates from
    it (OP_ACC_<wire>_TO_F32); unfused mode quantises locally and sends the narrow bytes with a plain isend.  The all-gather
    forwards the owner's quantised segment unchanged, so all ranks end with identical bits; the link carries
    count * wire_bytes * 2(n-1)/n bytes per rank instead of 4x / 2x that."""
    outs = _run_tring(world, count, f"c:{wire}:{fused}", piece, inflight)
    assert all(o["ok"] for o in outs), outs
    assert all(o["transport"] == "nvl" for o in outs)
    assert len({o["digest"] for o in outs}) == 1, "ranks disagree on the result"
    wes = 2 if wire == "bf16" else 1
    seg = -(-count // world)
    for o in outs:     # what left each rank: 2(n-1) segments in the wire format (segments are padded to 64 elements)
        assert o["stats"]["bytes_sent"] <= 2 * (world - 1) * (seg + 64) * wes
        assert o["stats"]["bytes_sent"] >= 2 * (world - 1) * (seg - 64 * world) * wes * 0.9


@pytest.mark.parametrize("impl", ["BASIC", "TOKIO"])
def test_transport_ring_compressed_allreduce_over_tcp(impl):
    """The same compressed all-reduce between hosts: the NVLink transport off, the narrow bytes travel over the TCP streams
    (unfused mode: quantise into the wire mirror, plain isend) — where a 4x smaller message pays most."""
    outs = _run_tring(3, 70001, "c:e4m3:0", 8192, 8, extra_env={"BNET_NVL": "0", "TRING_WIRE_HOST": "1", "BNET_IMPLEMENT": impl})
    assert all(o["ok"] for o in outs), outs
    assert all(o["transport"].startswith("tcp") for o in outs), outs
    assert len({o["digest"] for o in outs}) == 1


def _run_tmesh(world, count, idt, odt, piece, inflight, timeout=180, algo="one-shot", inplace=False, env_extra=None, mem="device"):
    import json
    import subprocess
    import sys
    import tempfile

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, BNET_FAKE_CUDA="1", BNET_NVL="1", PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    env.update(env_extra or {})
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, os.path.join(root, "tests", "tmesh_worker.py"), str(r), str(world), d, str(count),
                                   idt, odt, str(piece), str(inflight), "2", algo, "1" if inplace else "0", mem], env=env,
                                  stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
                 for r in range(world)]
        outs = []
        for p in procs:
            try:
                o, e = p.communicate(timeout=timeout)
            except subprocess.TimeoutExpired:
                for q in procs:
                    q.kill()
                raise
            assert p.returncode == 0, e[-3000:]
            outs.append(json.loads([ln for ln in o.splitlines() if ln.startswith("{")][-1]))
    return outs


@pytest.mark.parametrize("world,count,idt,odt,piece,inflight", [
    (2, 1 << 16, "f32", "f32", 16384, 4), (3, 100003, "bf16", "f32", 8192, 8), (4, 1 << 17, "bf16", "bf16", 65536, 8),
    (5, 7, "f32", "f32", 4096, 2), (8, 50000, "bf16", "f32", 16384, 8)])
def test_transport_mesh_oneshot_allreduce(world, count, idt, odt, piece, inflight):
    """The latency-optimal companion of the ring: a full mesh of plugin connections, ONE network step — every rank's
    kernel accumulates its input into every peer's output (isend_op(OP_RED_ADD_* / OP_ACC_BF16_TO_F32)), after a local
    pass initialised the output with the rank's own contribution.  Exact against the closed-form sum; the input is intact."""
    outs = _run_tmesh(world, count, idt, odt, piece, inflight)
    assert all(o["ok"] for o in outs), outs
    assert all(o["transport"] == "nvl" for o in outs)
    ies = 4 if idt == "f32" else 2
    assert all(o["stats"]["bytes_sent"] == (world - 1) * count * ies for o in outs), outs


@pytest.mark.parametrize("world,count,idt,odt,piece,inflight,inplace", [
    (2, 1 << 16, "f32", "f32", 16384, 4, False), (3, 100003, "bf16", "f32", 8192, 8, False), (4, 1 << 17, "bf16", "bf16", 65536, 8, True),
    (5, 7, "f32", "f32", 4096, 2, False), (8, 50000, "f32", "f32", 16384, 8, True), (8, 300, "bf16", "bf16", 4096, 2, False)])
def test_transport_mesh_twoshot_allreduce(world, count, idt, odt, piece, inflight, inplace):
    """The bandwidth-optimal shape on a switch, two network steps for any world size: every peer's kernel accumulates its
    part of slice r into rank r's output (fused isend), then the owner copies the finished slice to everybody.  Exact against
    the closed-form sum, in place or out of place, with slices that are short or empty (count < world * 64)."""
    outs = _run_tmesh(world, count, idt, odt, piece, inflight, algo="two-shot", inplace=inplace)
    assert all(o["ok"] for o in outs), outs
    assert all(o["transport"] == "nvl" for o in outs)
    ies, oes = (4 if idt == "f32" else 2), (4 if odt == "f32" else 2)
    seg = -(-(-(-count // world)) // 64) * 64
    sl = [max(0, min(count, (r + 1) * seg) - min(count, r * seg)) for r in range(world)]
    # rank r sends its part of every other slice (input type) and its own finished slice to every peer (output type)
    assert all(o["stats"]["bytes_sent"] == (sum(sl) - sl[r]) * ies + (world - 1) * sl[r] * oes for r, o in enumerate(outs)), outs


@pytest.mark.parametrize("name,env,transport", [
    ("tcp-basic", {"BNET_NVL": "0", "BNET_FAKE_CUDA": "0"}, "tcp-threads"),
    ("tcp-async", {"BNET_NVL": "0", "BNET_FAKE_CUDA": "0", "BAGUA_NET_IMPLEMENT": "TOKIO"}, "tcp-async"),
    ("shm", {"BNET_NVL": "1", "BNET_FAKE_CUDA": "0"}, "nvl")])
@pytest.mark.parametrize("world,count,idt,odt,inplace", [(3, 100003, "f32", "f32", True), (4, 70000, "bf16", "f32", False),
                                                          (5, 300, "bf16", "bf16", True), (2, 1 << 18, "f32", "f32", False)])
def test_transport_mesh_twoshot_on_host_memory_over_any_transport(name, env, transport, world, count, idt, odt, inplace):
    """Host memory is all-reduced with the same two-shot schedule over multi-stream TCP (both backends) and the same-host
    shared-memory ring: no fused isend there, the reduce-scatter pieces land in a staging area and are added on the host."""
    outs = _run_tmesh(world, count, idt, odt, 16384, 8, algo="two-shot", inplace=inplace, env_extra=env, mem="host")
    assert all(o["ok"] for o in outs), outs
    assert all(o["transport"] == transport for o in outs), [o["transport"] for o in outs]


# (torch's gloo process group and its OpenMP tensor kernels are not instrumented: ThreadSanitizer reports races inside
#  libtorch_cpu.so for this one; the same all-reduce without torch is test_transport_mesh_twoshot_on_host_memory_over_any_transport)
@pytest.mark.skipif("tsan" in os.environ.get("LD_PRELOAD", ""), reason="libtorch (gloo, OpenMP) under ThreadSanitizer")
@pytest.mark.parametrize("env,transport", [({"BNET_NVL": "0"}, "tcp-threads"), ({"BNET_NVL": "1"}, "nvl")])
def test_transport_mesh_torch_api_on_host_tensors(env, transport):
    """TransportMesh (the torch-facing wrapper) on CPU tensors: torch.distributed / gloo only exchanges the handles, the
    all-reduce rides the plugin's connections."""
    import json
    import socket
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    s_ = socket.socket()
    s_.bind(("127.0.0.1", 0))
    port = s_.getsockname()[1]
    s_.close()
    world = 3
    procs = []
    for r in range(world):
        e = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), BNET_FAKE_CUDA="0",
                 PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
        e.update(env)
        procs.append(subprocess.Popen([sys.executable, os.path.join(root, "tests", "tmesh_torch_worker.py")], env=e, stdout=subprocess.PIPE,
                                      stderr=subprocess.PIPE, text=True))
    for p in procs:
        try:
            o, err = p.communicate(timeout=180)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        assert p.returncode == 0, err[-3000:]
        d = json.loads([ln for ln in o.splitlines() if ln.startswith("{")][-1])
        assert d["ok"] and d["transport"] == transport, d


@pytest.mark.parametrize("seed", [11, 23, 37, 41, 59, 67])
def test_transport_mesh_randomized(seed):
    """Random world size, element count (including counts below one slice per rank), piece size, window, type pair,
    algorithm and placement: the sums must be exact every time."""
    import random

    rng = random.Random(seed)
    world = rng.choice([2, 3, 4, 5, 6, 7])
    count = rng.choice([1, 63, 64, 65, 1000, 4097, 65536 + rng.randrange(0, 5000), rng.randrange(100000, 400000)])
    algo = rng.choice(["one-shot", "two-shot"])
    idt, odt = rng.choice([("f32", "f32"), ("bf16", "bf16"), ("bf16", "f32")])
    inplace = algo == "two-shot" and idt == odt and rng.random() < 0.5
    piece, inflight = rng.choice([4096, 8192, 65536, 1 << 20]), rng.choice([1, 2, 8, 32])
    outs = _run_tmesh(world, count, idt, odt, piece, inflight, algo=algo, inplace=inplace)
    assert all(o["ok"] for o in outs), (world, count, algo, idt, odt, inplace, piece, inflight, outs)


@pytest.mark.parametrize("world,ver,count,dt,lib,mem,env", [
    (2, 8, 70000, "f32", "-", "dev", {}), (4, 6, 5000, "bf16", "-", "dev", {}), (3, 10, 33, "f32", "libnccl-net-bnetx.so", "dev", {}),
    (8, 8, 200000, "bf16", "-", "dev", {}),
    # host buffers (what NCCL hands a plugin without GPUDirect), over multi-stream TCP and the shared-memory ring
    (3, 8, 50000, "f32", "-", "host", {"BNET_NVL": "0", "BNET_FAKE_CUDA": "0"}),
    (4, 8, 30000, "bf16", "-", "host", {"BNET_NVL": "0", "BNET_FAKE_CUDA": "0", "BAGUA_NET_IMPLEMENT": "TOKIO"}),
    (2, 6, 100000, "f32", "-", "host", {"BNET_NVL": "1", "BNET_FAKE_CUDA": "0"})])
def test_collnet_table_allreduces_like_nccl_would_drive_it(world, ver, count, dt, lib, mem, env):
    """ncclCollNetPlugin_vN (csrc/plugin/collnet.cc): listen / connect(handles, nranks, rank) / regMr / iallreduce / test /
    iflush through the exported table, several all-reduces queued per rank and tested out of order; exact sums; sum of
    fp32 / bf16 on device memory (fused isends over the emulated NVLink transport) or host memory (TCP, shared memory)."""
    import json
    import subprocess
    import sys
    import tempfile

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    extra_env = env
    env = dict(os.environ, BNET_FAKE_CUDA="1", BNET_NVL="1", BNET_COLLNET="1",
               PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    env.update(extra_env)
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, os.path.join(root, "tests", "collnet_worker.py"), str(r), str(world), d, str(ver),
                                   str(count), dt, lib, mem], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
                 for r in range(world)]
        outs = []
        for p in procs:
            try:
                o, e = p.communicate(timeout=180)
            except subprocess.TimeoutExpired:
                for q in procs:
                    q.kill()
                raise
            assert p.returncode == 0, e[-3000:]
            outs.append(json.loads([ln for ln in o.splitlines() if ln.startswith("{")][-1]))
    for o in outs:
        assert o["ok"] and o["name"] == "BNet" and o["ndev"] >= 1 and o["bad_type_refused"], o
        assert o["ptr_support"] == (3 if env.get("BNET_FAKE_CUDA") == "1" else 1), o      # host always, device memory when CUDA is usable
        assert o["support"] == {"sum_this_type": True, "max": False, "int32": False}, o


def test_collnet_table_is_silent_unless_asked_for():
    """Without BNET_COLLNET=1 the table reports no devices: NCCL drops it at init and the net path is all it sees."""
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = {k: v for k, v in os.environ.items() if k != "BNET_COLLNET"}
    env.update(BNET_FAKE_CUDA="1", PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    code = ("from bagua_net_b200.utils.abi import CollNetPlugin\n"
            "p = CollNetPlugin(8); p.init(); print('ndev', p.devices())")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "ndev 0" in out.stdout, out.stderr[-2000:]


def test_nccl_tuner_plugin_picks_the_protocol_by_size():
    """ncclTunerPlugin_v3/_v4 inside the net plugin library (csrc/plugin/tuner.cc): over this transport LL for tiny messages,
    Simple above, LL128 never — and no opinion at all when the device path is off."""
    import json
    import subprocess
    import sys

    code = r'''
import ctypes as C, json, os
from bagua_net_b200.utils.abi import NetPlugin
from bagua_net_b200.utils.native import load
lib = load()
NetPlugin(8).init()                      # the net plugin's init ran in this process (NCCL does that before the tuner's)
LOG = C.c_void_p
class T4(C.Structure):
    _fields_ = [("name", C.c_char_p), ("init", C.CFUNCTYPE(C.c_int, C.c_size_t, C.c_size_t, LOG, C.POINTER(C.c_void_p))),
                ("getCollInfo", C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_size_t, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int))),
                ("destroy", C.CFUNCTYPE(C.c_int, C.c_void_p))]
class T3(C.Structure):
    _fields_ = [("name", C.c_char_p), ("init", C.CFUNCTYPE(C.c_int, C.c_size_t, C.c_size_t, LOG, C.POINTER(C.c_void_p))),
                ("getCollInfo", C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_size_t, C.c_int, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int))),
                ("destroy", C.CFUNCTYPE(C.c_int, C.c_void_p))]
out = {}
for ver, T in ((4, T4), (3, T3)):
    t = T.in_dll(lib, f"ncclTunerPlugin_v{ver}")
    ctx = C.c_void_p()
    assert t.init(8, 1, None, C.byref(ctx)) == 0
    res = {}
    for nbytes in (64, 8192, 8193, 1 << 20):
        table = (C.c_float * 21)(*([10.0] * 21))          # 7 algorithms x 3 protocols
        table[3 * 4 + 0] = -1.0                            # NCCL does not offer algorithm 4 with LL
        nch = C.c_int(0)
        args = [ctx, 4, nbytes, 1, C.cast(table, C.c_void_p), 7, 3] + ([0] if ver == 4 else []) + [C.byref(nch)]
        assert t.getCollInfo(*args) == 0
        res[nbytes] = [round(v, 1) for v in table]
    assert t.destroy(ctx) == 0
    out[ver] = res
print(json.dumps({"name": T4.in_dll(lib, "ncclTunerPlugin_v4").name.decode(), "out": out}))
'''
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for fake, active in (("1", True), ("0", False)):
        env = dict(os.environ, BNET_FAKE_CUDA=fake, BNET_NVL="1", PYTHONPATH=root)
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
        assert r.returncode == 0, r.stderr[-3000:]
        d = json.loads(r.stdout.splitlines()[-1])
        assert d["name"] == "BNet"
        for ver in ("4", "3"):
            small, edge, above, big = (d["out"][ver][k] for k in ("64", "8192", "8193", "1048576"))
            if not active:
                assert small == big == [10.0] * 12 + [-1.0] + [10.0] * 8      # no device path: the table is left alone
                continue
            for row in range(7):
                ll, ll128, simple = (small[3 * row + p] for p in range(3))
                assert ll128 == -1.0
                assert (ll, simple) == ((10.0, -1.0) if row != 4 else (-1.0, 10.0))   # LL where offered, else Simple stays
                assert edge[3 * row:3 * row + 3] == small[3 * row:3 * row + 3]
                assert above[3 * row:3 * row + 3] == [-1.0, -1.0, 10.0] and big[3 * row:3 * row + 3] == [-1.0, -1.0, 10.0]
    # BNET_COLLNET=1: wherever NCCL offers a CollNet algorithm (rows 2 and 3, Simple not "ignore") it is made the cheapest
    env = dict(os.environ, BNET_FAKE_CUDA="1", BNET_NVL="1", BNET_COLLNET="1", PYTHONPATH=root)
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr[-3000:]
    d = json.loads(r.stdout.splitlines()[-1])
    for ver in ("4", "3"):
        big = d["out"][ver]["1048576"]
        assert big[3 * 2 + 2] == 0.0 and big[3 * 3 + 2] == 0.0 and big[3 * 1 + 2] == 10.0 and big[3 * 0 + 2] == 10.0, big

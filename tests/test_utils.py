"""Unit tests of the OS utilities — same cases as the reference's only unit tests
(reference: src/utils.rs:263-314 test_parse / test_socket_handle / test_chunks) plus the
NIC-filter syntax and chunking invariants SURVEY.md §4 asks for."""
import json
import os
import subprocess
import time
import sys

import pytest

from bagua_net_b200 import utils

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_parse_user_pass_addr():
    assert utils.parse_user_pass_and_addr("nagle:1984@127.0.0.1:9090") == ("nagle", "1984", "127.0.0.1:9090")
    assert utils.parse_user_pass_and_addr("127.0.0.1:9090") == ("", "", "127.0.0.1:9090")
    assert utils.parse_user_pass_and_addr("") is None
    assert utils.parse_user_pass_and_addr("has space:1") is None


def test_socket_handle_roundtrip():
    # sockaddr -> 64-byte NCCL handle -> sockaddr (reference test_socket_handle: 127.0.0.1:8123)
    assert utils.sockaddr_roundtrip("127.0.0.1:8123") == "127.0.0.1:8123"
    # the reference truncates IPv6 at the FFI (src/lib.rs:157-158); ours fits
    assert utils.sockaddr_roundtrip("[fe80::1]:4242") == "[fe80::1]:4242"


def test_chunks_reference_cases():
    assert utils.chunk_count(1024, 1, 20) == 20
    assert utils.chunk_count(1024, 1000, 20) == 2


@pytest.mark.parametrize("total", [1, 15, 16, 4097, 1 << 20, (1 << 20) + 1, 123456789])
@pytest.mark.parametrize("minc", [1, 4096, 65535, 1 << 20])
@pytest.mark.parametrize("n", [1, 2, 3, 8])
def test_chunk_invariants(total, minc, n):
    cs = utils.chunk_size(total, minc, n)
    assert cs >= minc and cs * n >= total
    cnt = utils.chunk_count(total, minc, n)
    assert 1 <= cnt <= n                          # never more chunks than streams
    assert (cnt - 1) * cs < total <= cnt * cs     # both ends compute the same split


def test_if_filter_syntax():
    f = utils.if_filter_accepts
    assert not f("^docker,lo", "lo") and not f("^docker,lo", "docker0") and f("^docker,lo", "eth0")
    assert f("eth", "eth0") and f("eth", "eth1") and not f("eth", "ib0")      # prefix include
    assert f("=eth0", "eth0") and not f("=eth0", "eth01")                      # exact
    assert f("eth0,ib", "ib3") and not f("eth0,ib", "enp1s0")
    assert f("^=lo", "lo0") and not f("^=lo", "lo")


def test_find_interfaces_falls_back_to_loopback():
    env = dict(os.environ, NCCL_SOCKET_IFNAME="^docker,eth,en,ib,wl,ifb,veth,br")
    code = ("import json; from bagua_net_b200 import utils; print(json.dumps(utils.find_interfaces()))")
    env["PYTHONPATH"] = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, check=True).stdout
    # explicit user filter that excludes everything -> empty list, no silent fallback
    assert isinstance(json.loads(out), list)
    devs = utils.find_interfaces("lo")
    assert [d["name"] for d in devs] == ["lo"] and devs[0]["loopback"]
    assert devs[0]["speed"] == 10000          # default when sysfs has no speed (reference utils.rs:8)
    assert utils.find_interfaces("=doesnotexist0") == []
    v4 = utils.find_interfaces("lo", 2)
    assert v4 and v4[0]["addr"].startswith("127.0.0.1")


def test_base64_for_basic_auth():
    assert utils.base64("user:pass") == "dXNlcjpwYXNz"
    assert utils.base64("a") == "YQ==" and utils.base64("ab") == "YWI=" and utils.base64("") == ""


def test_config_env_aliases():
    env_code = "from bagua_net_b200 import utils; import json; print(json.dumps(utils.config()))"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def cfg(**env):
        e = {k: v for k, v in os.environ.items() if not k.startswith(("BNET_", "BAGUA_NET_"))}
        e.update(env, PYTHONPATH=root)
        return json.loads(subprocess.run([sys.executable, "-c", env_code], env=e, capture_output=True, text=True,
                                         check=True).stdout)

    d = cfg()
    assert d["implement"] == "BASIC" and d["nstreams"] == 2 and d["min_chunksize"] == 1048576   # reference defaults
    d = cfg(BAGUA_NET_IMPLEMENT="tokio")
    assert d["implement"] == "TOKIO" and d["min_chunksize"] == 65535
    d = cfg(BAGUA_NET_NSTREAMS="8", BAGUA_NET_MIN_CHUNKSIZE="4096", RANK="3")
    assert d["nstreams"] == 8 and d["min_chunksize"] == 4096 and d["rank"] == 3
    d = cfg(BNET_NSTREAMS="4", BAGUA_NET_NSTREAMS="8")          # BNET_* wins over the legacy name
    assert d["nstreams"] == 4
    d = cfg(BAGUA_NET_NSTREAMS="banana")                          # malformed: default, no abort
    assert d["nstreams"] == 2


def test_device_kernel_bodies_on_an_emulated_grid():
    """csrc/cuda/nn_body.cuh compiled by g++ and walked block by block, thread by thread (csrc/tests/nn_emu_test.cc):
    the row walk, batch tails, pool index coding and bias-gradient sums of the sm_90a kernels, without a GPU."""
    import subprocess

    import bagua_net_b200

    root = bagua_net_b200.REPO_ROOT
    # fused layer kernels; transport executor (copy/reduce/cast/fp8); wgmma linear (tiling, TMA boxes, epilogues)
    for name in ("nn_emu_test", "exec_emu_test", "tc_emu_test"):
        subprocess.run(["make", "-s", f"build/tests/{name}"], cwd=root, check=True, capture_output=True)
        r = subprocess.run([os.path.join(root, "build", "tests", name)], capture_output=True, text=True)
        assert r.returncode == 0 and "passed" in r.stdout, r.stdout[-2000:]


def test_doctor_reports_a_usable_setup_on_cpu():
    import io

    from bagua_net_b200 import doctor

    buf = io.StringIO()
    rc = doctor.run(out=buf)
    text = buf.getvalue()
    assert rc == 0, text
    assert "ncclNet tables exported: v3 v4 v5 v6 v7 v8" in text and "NCCL_NET_PLUGIN=bnet" in text


def test_bench_clock_sampler_with_a_stubbed_nvml(monkeypatch):
    """bench.py samples SM clocks / throttle reasons through NVML every 10 ms inside the timed region; here NVML is a
    stub (no GPU), on the H100 it is the real library and nvidia-smi stays as the fallback."""
    import importlib.util
    import time
    import types

    fake = types.ModuleType("pynvml")
    fake.NVML_CLOCK_SM = 1
    fake.nvmlInit = lambda: None
    fake.nvmlDeviceGetHandleByIndex = lambda i: i
    fake.nvmlDeviceGetMaxClockInfo = lambda h, c: 1965
    fake.nvmlDeviceGetClockInfo = lambda h, c: 1950
    fake.nvmlDeviceGetCurrentClocksThrottleReasons = lambda h: 0x4 | 0x1      # sw_power_cap + gpu idle
    monkeypatch.setitem(sys.modules, "pynvml", fake)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(root, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    s = mod.ClockSampler(0)
    s.start()
    time.sleep(0.15)
    out = s.stop()
    assert out["sm_mhz"] == 1950.0 and out["sm_max_mhz"] == 1965.0 and out["samples"] >= 5
    assert out["reasons"] == ["sw_power_cap"]


def test_symmcomm_tensor_collectives_logic_with_emulated_ranks():
    """all_reduce / broadcast / all_gather / reduce_scatter on ordinary tensors are compositions of the heap kernels,
    the barrier kernel and peer mappings (bagua_net_b200/parallel/comm.py).  Here the heap is CPU memory, the ranks are
    threads, the barrier is a threading.Barrier and the all-reduce kernel is a stub — what is checked is the staging,
    chunking, padding and slicing logic, with a stage small enough to force several chunks."""
    import threading

    import torch

    from bagua_net_b200.parallel.comm import SymmComm

    world = 4
    bar = threading.Barrier(world)
    comms = []
    for r in range(world):
        c = object.__new__(SymmComm)
        c.world, c.rank = world, r
        c._stage_buf = torch.zeros(16 * world * 40, dtype=torch.uint8)     # 2560 bytes: 640 floats per chunk
        c.launches = 0
        comms.append(c)
    red_lock = threading.Lock()
    pending = {}

    for c in comms:
        def peer_tensor(t, peer, c=c):
            off = t.data_ptr() - c._stage_buf.data_ptr()
            nbytes = t.numel() * t.element_size()
            return comms[peer]._stage_buf[off:off + nbytes].view(t.dtype).view(t.shape)

        def barrier(channel=2, stream=None):
            bar.wait()

        def all_reduce(st, op="sum", algo="auto", stream=None, c=c):
            assert st.numel() * st.element_size() % (16 * world) == 0, "all-reduce quantum violated"
            bar.wait()
            with red_lock:
                key = st.numel()
                pending.setdefault(key, []).append(st)
            bar.wait()
            if c.rank == 0:
                total = torch.stack([p.clone().float() for p in pending[st.numel()]]).sum(0)
                for p in pending[st.numel()]:
                    p.copy_(total.to(p.dtype))
                pending.clear()
            bar.wait()
            return st

        c.peer_tensor, c.barrier, c.all_reduce = peer_tensor, barrier, all_reduce

    inputs = [torch.arange(3001, dtype=torch.float32) * (r + 1) for r in range(world)]
    out = [None] * world
    errs = []

    def run(r):
        try:
            c = comms[r]
            res = {}
            res["ar"] = c.all_reduce_tensor(inputs[r].clone())
            b = inputs[r].clone()
            c.broadcast_tensor(b, src=2)
            res["bc"] = b
            res["ag"] = c.all_gather_tensor(inputs[r][:1501])
            res["rs"] = c.reduce_scatter_tensor(inputs[r][:3000])
            res["nc"] = c.all_reduce_tensor(torch.arange(35, dtype=torch.float32).view(5, 7).t() * (r + 1))   # non-contiguous
            out[r] = res
        except Exception as e:      # noqa: BLE001
            errs.append(repr(e))
            bar.abort()

    ths = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    [t.start() for t in ths]
    [t.join(60) for t in ths]
    assert not errs, errs
    total = sum(inputs)
    for r in range(world):
        assert torch.equal(out[r]["ar"], total)
        assert torch.equal(out[r]["bc"], inputs[2])
        assert torch.equal(out[r]["ag"], torch.stack([i[:1501] for i in inputs]))
        assert torch.equal(out[r]["rs"], total[:3000].view(world, -1)[r])
        assert torch.equal(out[r]["nc"], torch.arange(35, dtype=torch.float32).view(5, 7).t() * 10)


def test_ddp_bucket_plan_invariants():
    """Flat-buffer layout of the DDP engine (bagua_net_b200/parallel/ddp.py::plan_buckets)."""
    import random

    from bagua_net_b200.parallel.ddp import plan_buckets

    rnd = random.Random(3)
    for world in (1, 2, 4, 8):
        for es in (2, 4):
            for bucket_mb in (0.01, 0.25, 64.0):
                numels = [rnd.choice([1, 3, 64, 1000, 4096, 25088 * 16, 512 * 512 * 9]) for _ in range(rnd.randint(1, 40))]
                plan, total = plan_buckets(numels, es, world, bucket_mb)
                quantum = 16 * world // es * 8
                seen, end = [], 0
                for start, numel, members in plan:
                    assert start == end and numel % quantum == 0 and numel > 0
                    assert (numel // world) * es % 16 == 0                 # every rank's shard is whole 16-byte vectors
                    pos = start
                    for pi, off in members:
                        assert off >= pos and off % 8 == 0 and off + numels[pi] <= start + numel
                        pos = off + numels[pi]
                        seen.append(pi)
                    cap = int(bucket_mb * (1 << 20)) // es
                    assert len(members) == 1 or sum((numels[pi] + 7) // 8 * 8 for pi, _ in members) <= cap + quantum
                    end = start + numel
                assert total == end
                assert seen == list(reversed(range(len(numels))))           # reverse registration order, nothing lost
    # the flagship: VGG16's 32 tensors with 64 MB buckets
    vgg = [64 * 3 * 9, 64, 64 * 64 * 9, 64, 128 * 64 * 9, 128, 128 * 128 * 9, 128, 256 * 128 * 9, 256, 256 * 256 * 9, 256,
           256 * 256 * 9, 256, 512 * 256 * 9, 512, 512 * 512 * 9, 512, 512 * 512 * 9, 512, 512 * 512 * 9, 512, 512 * 512 * 9, 512,
           512 * 512 * 9, 512, 25088 * 4096, 4096, 4096 * 4096, 4096, 4096 * 1000, 1000]
    plan, total = plan_buckets(vgg, 2, 8, 64.0)
    assert sum(vgg) <= total < sum(vgg) + 40 * 1024 and len(plan) >= 3


def _cutlass_include():
    import glob
    import site

    for sp in site.getsitepackages():
        for cand in glob.glob(os.path.join(sp, "*", "data", "cutlass", "include")) + \
                glob.glob(os.path.join(sp, "*", "3rdparty", "cutlass", "include")):
            if os.path.exists(os.path.join(cand, "cute", "arch", "mma_sm90_desc.hpp")):
                return cand
    return None


def test_tcgen05_descriptors_match_cute_and_plans_are_sane():
    """The wgmma linear kernel (csrc/cuda/tc_gemm.cu) packs its shared-memory descriptors by hand;
    csrc/tests/tc_desc_test.cc compares them with the CuTe bit-field definitions and checks the tiling plans."""
    inc = _cutlass_include()
    if inc is None:
        pytest.skip("no CUTLASS headers with sm90 support in this environment")
    from bagua_net_b200 import LIB_DIR, LIB_NAME
    from bagua_net_b200.utils.native import load

    load()
    exe = os.path.join(ROOT, "build", "tests", "tc_desc_test")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-std=c++17", "-O1", f"-I{inc}", f"-I{ROOT}/include", "-I/usr/local/cuda/include",
                    os.path.join(ROOT, "csrc", "tests", "tc_desc_test.cc"), "-ldl", "-o", exe], check=True, timeout=300)
    r = subprocess.run([exe, os.path.join(LIB_DIR, LIB_NAME)], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr


def test_tc_linear_python_plan_and_gating(monkeypatch):
    from bagua_net_b200.ops import tc_linear

    monkeypatch.delenv("BNET_TC", raising=False)
    assert tc_linear.enabled()                           # on unless BNET_TC=0 ...
    monkeypatch.setenv("BNET_TC", "0")
    assert not tc_linear.enabled()
    monkeypatch.delenv("BNET_TC", raising=False)
    assert not tc_linear.trusted()                       # ... and still only trusted after its self-check passed on a GPU
    p = tc_linear.plan(32, 4096, 25088)                  # VGG16 fc1 at the flagship batch: weights fill the accumulator rows
    assert p["swap"] == 1 and p["bn"] == 32 and p["grid_y"] == 32 and p["k_blocks"] == 392
    p = tc_linear.plan(4096, 4096, 4096, reduce=True, splits=4)
    assert p["swap"] == 0 and p["bn"] == 256 and p["grid_z"] == 4 and p["k_per_split"] == 16 and p["ctas"] == 33
    assert p["smem_bytes"] + 1024 <= 227 * 1024
    with pytest.raises(ValueError):
        tc_linear.plan(32, 64, 100)
    assert tc_linear.self_check() is False or __import__("torch").cuda.is_available()   # no GPU here: a clean False


def test_tc_self_check_runs_isolated_and_is_cached(monkeypatch, tmp_path):
    """The opt-in wgmma path is only trusted after its self-check passed in a CHILD process (a faulting kernel must not
    poison the trainer's CUDA context); the verdict is cached per library build and GPU model."""
    import glob

    import torch

    from bagua_net_b200.ops import tc_linear

    monkeypatch.setenv("BNET_CACHE_DIR", str(tmp_path))
    monkeypatch.setattr(torch.cuda, "get_device_name", lambda *a: "Fake H100")
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    assert tc_linear._isolated_self_check(timeout=120) is False        # no GPU in the child either: no verdict, nothing cached
    assert not glob.glob(str(tmp_path / "tc_self_check_*.json"))
    assert tc_linear._isolated_self_check(timeout=0.001) is False      # (a timeout — e.g. under a profiler — is no verdict either)
    # definitive outcomes are cached: the check ran and failed (exit 3), passed (exit 0), or the child died by a signal
    failing = "import sys; sys.exit(3)"
    import subprocess as sp
    import types

    calls = []

    def fake_run(cmd, **kw):
        calls.append(cmd[-1])
        return types.SimpleNamespace(returncode=fake_run.rc)

    monkeypatch.setattr(sp, "run", fake_run)
    for rc, want, cached in ((3, False, True), (-11, False, True), (1, False, False), (0, True, True)):
        fake_run.rc = rc
        tag = f"t_rc{abs(rc)}"
        assert tc_linear._isolated_self_check(timeout=5, check=failing, tag=tag) is want
        files = glob.glob(str(tmp_path / f"{tag}_*.json"))
        assert (len(files) == 1 and json.load(open(files[0]))["ok"] is want) if cached else not files, (rc, files)
    assert failing in calls[-1] and calls[-1].endswith("sys.exit(0 if ok else 3)")
    n = len(calls)
    assert tc_linear._isolated_self_check(timeout=5, check=failing, tag="t_rc0") is True and len(calls) == n   # cached: no child


def test_tc_conv_wgrad_plan_and_gating(monkeypatch, tmp_path):
    """The wgmma filter gradient: every VGG16 layer it accepts (batch 32) is cut into enough pixel slices to put 124+ CTAs
    on the 132 SMs of an H100 (the library plans for them when it sees no GPU) with one resident CTA each, within shared
    memory; and the kernel is only trusted after a self-check in a child process, with the verdict cached under its own name."""
    import glob

    import torch

    from bagua_net_b200.ops import tc_conv, tc_linear

    for cin, cout, hw in ((64, 64, 224), (64, 128, 112), (128, 128, 112), (128, 256, 56), (256, 256, 56), (256, 512, 28), (512, 512, 28),
                          (512, 512, 14)):
        p = tc_conv.wgrad_plan(32, hw, hw, cin, cout)
        assert 124 <= p["ctas"] * p["grid_z"] <= 132, (cin, cout, hw, p)
        assert p["k_blocks"] == 32 * hw * hw // 64 and p["k_per_split"] * p["grid_z"] >= p["k_blocks"]          # exact 64-pixel patches
        assert (p["grid_z"] - 1) * p["k_per_split"] < p["k_blocks"]                                              # no empty slice
        assert p["grid_x"] * p["bn"] >= 9 * cin and p["grid_y"] * 128 >= cout and p["smem_bytes"] + 1024 <= 227 * 1024
        assert p["grid_x"] * p["grid_y"] <= tc_conv._L().bnet_tc_conv3x3_wgrad_tiles(cin, cout)
    assert tc_conv.wgrad_plan(32, 28, 28, 512, 512, splits=1)["grid_z"] == 1
    assert tc_conv.wgrad_plan(32, 28, 28, 512, 512, splits=1)["ctas"] == 72
    with pytest.raises(ValueError):
        tc_conv.wgrad_plan(32, 224, 224, 3, 64)                      # the first layer stays with cuDNN
    # gating: off by switch, and without a passing child-process check
    monkeypatch.setenv("BNET_TC_WGRAD", "0")
    monkeypatch.setattr(tc_conv, "_wgrad_trusted", None)
    assert tc_conv.wgrad_trusted() is False
    monkeypatch.delenv("BNET_TC_WGRAD", raising=False)
    monkeypatch.setattr(tc_conv, "_wgrad_trusted", None)
    monkeypatch.setattr(tc_conv, "usable", lambda: True)
    monkeypatch.setenv("BNET_CACHE_DIR", str(tmp_path))
    monkeypatch.setattr(torch.cuda, "get_device_name", lambda *a: "Fake H100")
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    monkeypatch.delenv("BNET_TC_WGRAD_BN", raising=False)
    monkeypatch.delenv("BNET_TC_WGRAD_FIXUP", raising=False)
    import subprocess

    spawned, real_run = [], subprocess.run
    monkeypatch.setattr(subprocess, "run", lambda *a, **k: (spawned.append(1), real_run(*a, **k))[1])
    assert tc_conv.wgrad_trusted() is False                          # the child has no GPU either: not trusted, nothing cached
    monkeypatch.setattr(subprocess, "run", real_run)
    assert len(spawned) == 1                                         # ... and no verdict stops the ladder: one child, not four
    assert not glob.glob(str(tmp_path / "tc_wgrad_*self_check_*.json")) and "BNET_TC_WGRAD_BN" not in os.environ
    # verdict files as a GPU box would leave them: the default plan failed its check, the 128-column ladder step passed
    import hashlib

    import bagua_net_b200

    lib = os.path.join(bagua_net_b200.LIB_DIR, bagua_net_b200.LIB_NAME)
    key = f"{os.path.getmtime(lib):.0f}-{os.path.getsize(lib)}-Fake H100-{torch.version.cuda}"
    h = hashlib.sha1(key.encode()).hexdigest()[:16]
    json.dump({"ok": False}, open(tmp_path / f"tc_wgrad_self_check_{h}.json", "w"))
    json.dump({"ok": True}, open(tmp_path / f"tc_wgrad_bn128_self_check_{h}.json", "w"))
    monkeypatch.setattr(tc_conv, "_wgrad_trusted", None)
    assert tc_conv.wgrad_trusted() is True and os.environ.get("BNET_TC_WGRAD_BN") == "128"
    monkeypatch.delenv("BNET_TC_WGRAD_BN", raising=False)
    # further down the ladder: neither tile width passes with the in-kernel finish, the plain-reduce mode does
    json.dump({"ok": False}, open(tmp_path / f"tc_wgrad_bn128_self_check_{h}.json", "w"))
    json.dump({"ok": True}, open(tmp_path / f"tc_wgrad_nofix_self_check_{h}.json", "w"))
    monkeypatch.setattr(tc_conv, "_wgrad_trusted", None)
    assert tc_conv.wgrad_trusted() is True and os.environ.get("BNET_TC_WGRAD_FIXUP") == "0" and "BNET_TC_WGRAD_BN" not in os.environ
    monkeypatch.delenv("BNET_TC_WGRAD_FIXUP", raising=False)
    json.dump({"ok": False}, open(tmp_path / f"tc_wgrad_nofix_self_check_{h}.json", "w"))
    json.dump({"ok": False}, open(tmp_path / f"tc_wgrad_bn128_nofix_self_check_{h}.json", "w"))
    monkeypatch.setattr(tc_conv, "_wgrad_trusted", None)
    assert tc_conv.wgrad_trusted() is False and "BNET_TC_WGRAD_BN" not in os.environ and "BNET_TC_WGRAD_FIXUP" not in os.environ
    assert not glob.glob(str(tmp_path / "tc_self_check_*.json"))     # (the linear kernel's verdict is a different file)


# pure-PyTorch tests (no native code of ours involved): skipped under ThreadSanitizer, whose runtime reports races inside
# libtorch's own OpenMP convolution kernels (uninstrumented libgomp) — ci/run_sanitizers.sh is about OUR host engine
no_tsan = pytest.mark.skipif("tsan" in os.environ.get("LD_PRELOAD", ""), reason="libtorch CPU kernels under ThreadSanitizer")


@no_tsan
def test_conv_backward_composes_tcgen05_and_library_gradients(monkeypatch):
    """fused_nn._conv_backward asks the autotuner per gradient (input / filter) and per shape; whatever mix it answers, the
    pair that comes back must be the convolution's gradients, and a gradient nobody asked for is not computed."""
    import torch

    from bagua_net_b200.ops import fused_nn, tc_conv

    torch.manual_seed(0)
    x = torch.randn(2, 8, 6, 6).bfloat16().contiguous(memory_format=torch.channels_last)
    w = torch.randn(16, 8, 3, 3).bfloat16().contiguous(memory_format=torch.channels_last)
    gz = torch.randn(2, 16, 6, 6).bfloat16().contiguous(memory_format=torch.channels_last)
    ref_x, ref_w, _ = torch.ops.aten.convolution_backward(gz, x, w, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [True, True, False])
    calls = []

    def fake_dgrad(g, ww):
        calls.append("tc_dgrad")
        return torch.ops.aten.convolution_backward(g, x, ww, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [True, False, False])[0]

    def fake_wgrad(g, xx, splits=0, out=None):
        calls.append("tc_wgrad")
        r = torch.ops.aten.convolution_backward(g, xx, w, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [False, True, False])[1]
        if out is not None:
            out.copy_(r)
            return out
        return r

    monkeypatch.setattr(tc_conv, "conv3x3_dgrad", fake_dgrad)
    monkeypatch.setattr(tc_conv, "conv3x3_wgrad", fake_wgrad)
    for pick_x in ("tc", "cudnn"):
        for pick_w in ("tc", "cudnn"):
            for need_x in (True, False):
                monkeypatch.setattr(tc_conv, "choose", lambda kind, *a, _p=pick_x, **k: _p)
                monkeypatch.setattr(tc_conv, "choose_wgrad", lambda *a, _p=pick_w, **k: _p)
                calls.clear()
                gx, gw = fused_nn._conv_backward(gz, x, w, [1, 1], [1, 1], need_x)
                assert torch.equal(gw, ref_w), (pick_x, pick_w, need_x)
                assert (gx is None) if not need_x else torch.equal(gx, ref_x), (pick_x, pick_w, need_x)
                assert calls.count("tc_dgrad") == (1 if (need_x and pick_x == "tc") else 0), (calls, pick_x, pick_w, need_x)
                assert calls.count("tc_wgrad") == (1 if pick_w == "tc" else 0), (calls, pick_x, pick_w, need_x)
    # an engine registered a gradient slice for this filter: the kernel writes there, autograd gets a tensor over that memory
    from bagua_net_b200.ops import grad_target

    slot = torch.zeros(w.numel() + 8, dtype=torch.bfloat16)
    off = (-slot.data_ptr() // 2) % 8                                   # 16-byte aligned start inside the buffer
    dst = slot[off:off + w.numel()].view(16, 3, 3, 8).permute(0, 3, 1, 2)   # channels_last like the filter
    grad_target.register(w, dst)
    monkeypatch.setattr(tc_conv, "choose", lambda *a, **k: "cudnn")
    monkeypatch.setattr(tc_conv, "choose_wgrad", lambda *a, **k: "tc")
    gx, gw = fused_nn._conv_backward(gz, x, w, [1, 1], [1, 1], True)
    assert gw.data_ptr() == dst.data_ptr() and gw is not dst and torch.equal(gw, ref_w) and torch.equal(dst, ref_w)
    grad_target.unregister(w)
    assert grad_target.lookup(w) is None
    # anything but 3x3 / stride 1 / pad 1 never reaches the autotuner
    monkeypatch.setattr(tc_conv, "choose", lambda *a, **k: (_ for _ in ()).throw(AssertionError("asked")))
    monkeypatch.setattr(tc_conv, "choose_wgrad", lambda *a, **k: (_ for _ in ()).throw(AssertionError("asked")))
    w1 = torch.randn(16, 8, 1, 1).bfloat16().contiguous(memory_format=torch.channels_last)
    gx, gw = fused_nn._conv_backward(gz, x, w1, [1, 1], [0, 0], True)
    assert gx.shape == x.shape and gw.shape == w1.shape


def test_wgrad_self_check_can_be_given_the_callers_shapes(monkeypatch):
    from bagua_net_b200.ops import tc_conv

    monkeypatch.delenv("BNET_TC_WGRAD_CHECK_SHAPES", raising=False)
    assert tc_conv._extra_check_shapes() == ((), "")
    monkeypatch.setenv("BNET_TC_WGRAD_CHECK_SHAPES", "32,64,64,224;32,512,512,14;32,3,64,224;junk;32,64,128,0;32,512,512,14")
    shapes, sfx = tc_conv._extra_check_shapes()
    assert shapes == ((32, 64, 64, 224, 0), (32, 512, 512, 14, 0)) and len(sfx) == 9 and sfx.startswith("_")
    # what the child evaluates must be valid Python that extends the built-in list
    ns = {}
    exec(f"from bagua_net_b200.ops import tc_conv\nall_shapes = tc_conv.WGRAD_CHECK_SHAPES + {shapes!r}", ns)
    assert ns["all_shapes"][-1] == (32, 512, 512, 14, 0) and len(ns["all_shapes"]) == len(tc_conv.WGRAD_CHECK_SHAPES) + 2
    monkeypatch.setenv("BNET_TC_WGRAD_CHECK_SHAPES", "8,64,64,32")
    assert tc_conv._extra_check_shapes()[1] != sfx                     # another shape list, another verdict file


@no_tsan
def test_wgrad_self_check_body_runs(monkeypatch):
    """The child-process self-check of the filter gradient is what decides whether the kernel is ever used: its own Python
    must not be what fails.  Run its body on the CPU with the kernel replaced by the library's result (and by a wrong one)."""
    import torch

    from bagua_net_b200.ops import tc_conv, tc_linear

    state = {"scale": 1.0, "dirty": False}

    def fake_wgrad(gy, x, splits=0):
        w = torch.empty(gy.shape[1], x.shape[1], 3, 3, dtype=torch.bfloat16)
        ws, _ = tc_conv._wgrad_ws(gy.device, x.shape[1], gy.shape[1])
        if state["dirty"]:
            ws[0, 0] = 1.0
        ref = torch.ops.aten.convolution_backward(gy, x, w, None, [1, 1], [1, 1], [1, 1], False, [0, 0], 1, [False, True, False])[1]
        return (ref.float() * state["scale"]).to(torch.bfloat16)

    monkeypatch.setattr(tc_conv, "conv3x3_wgrad", fake_wgrad)
    monkeypatch.setattr(tc_conv, "_wgrad_scratch", {})
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(tc_linear, "last_error", lambda *a: 0)
    cpu, small = torch.device("cpu"), ((2, 64, 64, 6, 0), (1, 64, 128, 5, 2))
    assert tc_conv.self_check_wgrad(device=cpu, shapes=small) is True
    state["scale"] = 1.3
    assert tc_conv.self_check_wgrad(device=cpu, shapes=small) is False          # wrong numbers
    state["scale"], state["dirty"] = 1.0, True
    assert tc_conv.self_check_wgrad(device=cpu, shapes=small) is False          # scratch not handed back clean
    state["dirty"] = False
    monkeypatch.setattr(tc_conv, "_wgrad_scratch", {})
    monkeypatch.setattr(tc_linear, "last_error", lambda *a: 2)
    assert tc_conv.self_check_wgrad(device=cpu, shapes=small) is False          # the pipeline watchdog tripped
    assert len(tc_conv.WGRAD_CHECK_SHAPES) >= 6 and any(s[1] == 64 for s in tc_conv.WGRAD_CHECK_SHAPES)   # 128- and 256-column plans


def test_wgrad_autotuner_decisions(monkeypatch):
    """choose_wgrad: untrusted kernel, wrong results, a tripped watchdog or an exception keep cuDNN; otherwise the faster
    implementation wins; every verdict is cached per layer shape."""
    import torch

    from bagua_net_b200.ops import tc_conv, tc_linear

    w = torch.zeros(64, 64, 3, 3).bfloat16().contiguous(memory_format=torch.channels_last)
    good = torch.ones(64, 64, 3, 3)
    state = {"trusted": True, "tc": good, "watchdog": 0, "t": {"tc": 10.0, "lib": 20.0}}
    monkeypatch.setattr(tc_conv, "usable", lambda: True)
    monkeypatch.setattr(tc_conv, "wgrad_shape_ok", lambda a, b: True)
    monkeypatch.setattr(tc_conv, "wgrad_trusted", lambda: state["trusted"])
    monkeypatch.setattr(tc_conv, "mode", lambda: "auto")
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    monkeypatch.setattr(tc_linear, "last_error", lambda *a: state["watchdog"])

    def fake_wgrad(g, xx, splits=0):
        if isinstance(state["tc"], Exception):
            raise state["tc"]
        return state["tc"]

    monkeypatch.setattr(tc_conv, "conv3x3_wgrad", fake_wgrad)
    lib = lambda: good                                                     # noqa: E731
    monkeypatch.setattr(tc_conv, "_time_us", lambda fn, iters=5: state["t"]["lib"] if fn is lib else state["t"]["tc"])

    def decide(n):                                                         # a fresh shape (batch n) every time
        x = torch.zeros(n, 64, 4, 4).bfloat16().contiguous(memory_format=torch.channels_last)
        return tc_conv.choose_wgrad(torch.zeros_like(x), x, w, lib), ("wgrad", n, 4, 4, 64, 64)

    monkeypatch.setattr(tc_conv, "_choice", {})
    monkeypatch.setattr(tc_conv, "TIMINGS", {})
    pick, key = decide(1)
    assert pick == "tc" and tc_conv.TIMINGS[key] == {"tc": 10.0, "cudnn": 20.0}
    state["t"] = {"tc": 30.0, "lib": 20.0}
    assert decide(1)[0] == "tc"                                            # cached: not timed again
    assert decide(2)[0] == "cudnn"
    state["t"] = {"tc": 10.0, "lib": 20.0}
    state["tc"] = good * 1.5
    pick, key = decide(3)
    assert pick == "cudnn" and "differ" in tc_conv.TIMINGS[key]["error"]
    state["tc"], state["watchdog"] = good, 2
    pick, key = decide(4)
    assert pick == "cudnn" and "watchdog" in tc_conv.TIMINGS[key]["error"]
    state["watchdog"], state["tc"] = 0, RuntimeError("bnet_tc_conv3x3_wgrad: no kernel")
    pick, key = decide(5)
    assert pick == "cudnn" and "RuntimeError" in tc_conv.TIMINGS[key]["error"]
    state["tc"], state["trusted"] = good, False
    pick, key = decide(6)
    assert pick == "cudnn" and "not trusted" in tc_conv.TIMINGS[key]["error"]
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    state["trusted"] = True
    assert decide(7)[0] == "cudnn" and ("wgrad", 7, 4, 4, 64, 64) not in tc_conv._choice     # a capture decides nothing


def test_bench_child_jobs_are_bounded_and_fail_soft(monkeypatch, tmp_path):
    """The side measurements of bench.py (DDP arms, ResNet arms, transport collectives, the CollNet probe) are child
    processes: a result file is merged into the status, a child that fails or outlives its timeout costs that entry only."""
    import argparse
    import importlib.util

    spec = importlib.util.spec_from_file_location("bench_under_test3", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    monkeypatch.setenv("BNET_BENCH_LOG_DIR", str(tmp_path))
    monkeypatch.setenv("MASTER_PORT", "29500")
    monkeypatch.setenv("TORCHELASTIC_RUN_ID", "x")
    args = argparse.Namespace(model="vgg16", steps=20, batch=32, image=224, no_fused=False, no_graph=False)
    good = tmp_path / "good.py"
    good.write_text("import argparse, json, os, sys\n"
                    "a = argparse.ArgumentParser(); a.add_argument('--json'); a = a.parse_args()\n"
                    "assert os.environ['BNET_BENCH_CHILD'] == '1' and 'TORCHELASTIC_RUN_ID' not in os.environ\n"
                    "assert os.environ['MASTER_PORT'] == '29650' and 'BNET_BENCH_FUSED_VERDICT' not in os.environ\n"
                    "print('child log line')\n"
                    "open(a.json, 'w').write(json.dumps({'busbw': 123.0, 'exact': True}))\n")
    res = mod.run_child_arm("transport", args, 0, 2, 150, 30.0, model="coll", script=[str(good)])
    assert res["status"] == "ok" and res["busbw"] == 123.0 and res["exact"] is True and os.path.exists(res["log_path"])
    assert "child log line" in open(res["log_path"]).read()
    assert mod.run_child_arm("transport", args, 1, 2, 150, 30.0, model="coll", script=[str(good)]) is None     # only rank 0 reports
    bad = tmp_path / "bad.py"
    bad.write_text("import sys\nprint('boom: something failed')\nsys.exit(7)\n")
    res = mod.run_child_arm("collnet", args, 0, 2, 163, 30.0, model="probe", script=[str(bad)])
    assert res["status"] == "exit code 7" and any("boom" in ln for ln in res["log_tail"])
    slow = tmp_path / "slow.py"
    slow.write_text("import time\ntime.sleep(60)\n")
    t0 = time.time()
    res = mod.run_child_arm("collnet", args, 0, 2, 163, 1.0, model="probe", script=[str(slow)])
    assert res["status"].startswith("timeout") and time.time() - t0 < 20


def test_bench_isolated_self_check_classifies_child_outcomes(monkeypatch):
    """bench.py trusts the fused layer kernels only after their self-check ran in a child process: verdicts (exit 0 / 3,
    or death by signal) are final, anything else falls back to the in-process check."""
    import importlib.util
    import types

    spec = importlib.util.spec_from_file_location("bench_under_test2", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    seen = {}

    def fake_run(cmd, env=None, timeout=None, **kw):
        seen["env"], seen["code"] = env, cmd[-1]
        if fake_run.rc == "timeout":
            raise subprocess.TimeoutExpired(cmd, timeout)
        return types.SimpleNamespace(returncode=fake_run.rc)

    monkeypatch.setattr(mod.subprocess, "run", fake_run)
    monkeypatch.setenv("RANK", "3")
    monkeypatch.setenv("WORLD_SIZE", "8")
    for rc, want in ((0, True), (3, False), (-11, False), (-6, False), (4, None), (1, None), ("timeout", False)):
        fake_run.rc = rc
        assert mod.isolated_self_check("self_check", 5) is want, rc
    assert "RANK" not in seen["env"] and "WORLD_SIZE" not in seen["env"] and ROOT in seen["env"]["PYTHONPATH"]
    assert "set_device(5)" in seen["code"] and "fused_nn.self_check()" in seen["code"]
    compile(seen["code"], "<child>", "exec")
    # and for real, without a GPU: the child cannot even select a device -> "unrelated reason" -> None
    monkeypatch.undo()
    assert mod.isolated_self_check("self_check", 0, timeout=120) is None


def test_shell_scripts_parse():
    """Every shell script of the repo at least parses (the GPU session runner cannot be exercised without a GPU)."""
    import glob
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    scripts = sorted(glob.glob(os.path.join(root, "tools", "*.sh")) + glob.glob(os.path.join(root, "ci", "*.sh")))
    assert scripts
    for s in scripts:
        env = {k: v for k, v in os.environ.items() if k != "LD_PRELOAD"}       # (a sanitizer runtime preloaded into bash crashes it)
        r = subprocess.run(["bash", "-n", s], capture_output=True, text=True, env=env)
        assert r.returncode == 0, f"{s}: {r.stderr}"
    # the recipe names documented in the header of the session runner are the ones its case statement knows
    src = open(os.path.join(root, "tools", "gpu_session.sh")).read()
    header = [ln.split()[1] for ln in src.splitlines() if ln.startswith("#   ") and len(ln.split()) > 2 and ln[4] != " " and not ln.startswith("#   gpurun")]
    for name in header:
        assert f"{name})" in src or f"|{name})" in src or f"{name}|" in src, name


def test_plugin_environment_helper(monkeypatch):
    """What `python -m bagua_net_b200.utils.env` hands to NCCL: the plugin + tuner names, forced net transport, GDR, and the
    module-loading mode (eager by default; lazy on request; never overriding what the user exported)."""
    from bagua_net_b200.utils.env import nccl_plugin_env

    for k in ("CUDA_MODULE_LOADING", "CUDA_DEVICE_MAX_CONNECTIONS", "BNET_TUNER", "NCCL_BUFFSIZE"):
        monkeypatch.delenv(k, raising=False)
    e = nccl_plugin_env(force_net=True)
    assert e["NCCL_NET_PLUGIN"] == "bnet" and e["NCCL_NET"] == "BNet" and e["NCCL_TUNER_PLUGIN"] == "bnet"
    assert e["NCCL_P2P_DISABLE"] == "1" and e["NCCL_SHM_DISABLE"] == "1" and e["NCCL_NET_GDR_LEVEL"] == "SYS"
    import bagua_net_b200

    assert e["CUDA_MODULE_LOADING"] == "EAGER" and e["LD_LIBRARY_PATH"].split(os.pathsep)[0] == bagua_net_b200.LIB_DIR
    assert "CUDA_MODULE_LOADING" not in nccl_plugin_env(eager_modules=False)
    monkeypatch.setenv("CUDA_MODULE_LOADING", "LAZY")
    assert "CUDA_MODULE_LOADING" not in nccl_plugin_env()            # the user's choice stands
    monkeypatch.setenv("BNET_TUNER", "0")
    assert "NCCL_TUNER_PLUGIN" not in nccl_plugin_env()
    assert nccl_plugin_env(gdr=False)["BNET_GDR"] == "0"
    assert nccl_plugin_env(tuned=True)["NCCL_BUFFSIZE"] == str(32 << 20)
    assert "NCCL_TUNER_PLUGIN" not in nccl_plugin_env(plugin="bnetx")


def test_bench_headline_survives_hung_or_failing_optional_parts(tmp_path):
    """Once bench.py's timed region is over its number is printed whatever the optional measurements do: a watchdog (every rank
    runs the same timer) kills a child arm that is still running, prints the contract's JSON line from what is there — e2e and
    checksum included when they were finished — and ends the process with exit code 0; an exception that escapes main() after
    the headline takes the same exit."""
    script = tmp_path / "drive.py"
    script.write_text(
        "import argparse, importlib.util, os, subprocess, sys, time\n"
        f"spec = importlib.util.spec_from_file_location('bench_wd', {os.path.join(ROOT, 'bench.py')!r})\n"
        "mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)\n"
        "args = argparse.Namespace(model='vgg16', steps=20, warmup=5, batch=32, image=224, comm='bnet', child_json=None,\n"
        "                          resnet_deadline=300.0, resnet_timeout=90.0, arm_timeout=150.0, no_arms=False)\n"
        "extra = {}\n"
        "mod._HEADLINE.update({'extra': extra, 'args': args, 'world': 1, 'rank': 0, 'img_s': 7000.0, 'ms_step': 4.571,\n"
        "                      'clocks': {'sm_mhz': 1965, 'sm_max_mhz': 1965, 'reasons': []}, 'nlaunch': 1234, 'wall_ms': 4.6,\n"
        "                      'path': 'single', 'fused': True, 'graph_used': True, 'n_params': 138357544})\n"
        "mod._HEADLINE['e2e'] = {'value': 6990.0, 'unit': 'img/s', 'h2d_bytes_per_step': 9633792 + 256, 'd2h_bytes_per_step': 4}\n"
        "extra['allreduce_algo'] = 'single'\n"
        "if sys.argv[1] == 'hang':\n"
        "    os.environ['BNET_BENCH_HARD_DEADLINE'] = str(time.time() - mod._T0 + 1.5)\n"
        "    mod.arm_watchdog()\n"
        "    child = subprocess.Popen([sys.executable, '-c', 'import time; time.sleep(120)'])\n"
        "    mod._CHILDREN.append(child)\n"
        "    print(child.pid, file=sys.stderr, flush=True)\n"
        "    child.wait()\n"
        "    time.sleep(60)\n"
        "    sys.exit(9)\n"
        "else:\n"
        "    def boom():\n"
        "        raise RuntimeError('CUDA error: an illegal memory access was encountered')\n"
        "    mod._main = boom\n"
        "    sys.exit(mod.main())\n")
    for how in ("hang", "raise"):
        t0 = time.time()
        r = subprocess.run([sys.executable, str(script), how], capture_output=True, text=True, timeout=60)
        assert r.returncode == 0 and time.time() - t0 < 30, (how, r.returncode, r.stderr[-400:])
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
        assert len(lines) == 1, r.stdout
        out = json.loads(lines[0])
        assert out["metric"] == "vgg16_train_img_per_sec" and out["value"] == 7000.0 and out["n_gpus"] == 1
        assert out["steps"] == 20 and out["warmup"] == 5 and out["higher_is_better"] is True and out["scaling"] == "weak"
        assert out["gpu_launches"] == 1234 and out["e2e"]["value"] == 6990.0 and out["clocks"]["sm_mhz"] == 1965
        assert out["config"]["global_batch"] == 32 and out["extra"]["allreduce_algo"] == "single"
        assert ("watchdog" if how == "hang" else "illegal memory access") in out["extra"]["cut_short"]
        if how == "hang":           # the child arm that was still running is gone (its exact pid was killed)
            pid = int(r.stderr.split()[0])
            with pytest.raises(ProcessLookupError):
                for _ in range(50):
                    os.kill(pid, 0)
                    time.sleep(0.1)


def test_bench_failed_run_is_repeated_in_a_fresh_process_with_the_unproven_paths_off(tmp_path):
    """A 1-GPU run that fails before its timed region is over is repeated by a fresh process (a faulting kernel poisons the CUDA
    context) with the paths that have the least hardware mileage switched off — level by level, each level a superset of the one
    before; a multi-rank job and the reference arm are never repeated."""
    script = tmp_path / "drive.py"
    script.write_text(
        "import importlib.util, os, sys\n"
        f"spec = importlib.util.spec_from_file_location('bench_retry', {os.path.join(ROOT, 'bench.py')!r})\n"
        "mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)\n"
        "def fake():\n"
        "    lvl = os.environ.get('BNET_BENCH_SAFE_LEVEL', '0')\n"
        "    print('attempt', lvl, os.environ.get('BNET_DIRECT_GRADS'), os.environ.get('BNET_TC_WGRAD'), os.environ.get('BNET_TC'), flush=True)\n"
        "    if int(lvl) < int(sys.argv[1]):\n"
        "        raise RuntimeError('boom at level ' + lvl)\n"
        "    print('reason', os.environ.get('BNET_BENCH_SAFE_REASON'), flush=True)\n"
        "    return 0\n"
        "mod._main = fake\n"
        "sys.exit(mod.main())\n")
    env = {k: v for k, v in os.environ.items() if not k.startswith("BNET_") and k != "WORLD_SIZE"}
    r = subprocess.run([sys.executable, str(script), "2"], capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode == 0, r.stderr[-400:]
    assert [ln for ln in r.stdout.splitlines() if ln.startswith("attempt")] == [
        "attempt 0 None None None", "attempt 1 0 0 None", "attempt 2 0 0 0"]
    assert "reason RuntimeError: boom at level 1" in r.stdout
    r = subprocess.run([sys.executable, str(script), "3"], capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode != 0 and r.stdout.count("attempt") == 3 and "boom at level 2" in r.stderr      # the ladder is finite
    r = subprocess.run([sys.executable, str(script), "1"], capture_output=True, text=True, timeout=120, env=dict(env, WORLD_SIZE="2"))
    assert r.returncode != 0 and r.stdout.count("attempt") == 1                                         # multi-rank: no repeat

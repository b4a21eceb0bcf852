"""GPU tests (run on an H100 with `pytest -m gpu`).  Every kernel is compared against a plain
PyTorch fp32 reference of the same op.  Multi-GPU cases launch one process per GPU and are
skipped on a single-GPU box."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _torch():
    import torch

    assert torch.cuda.is_available(), "GPU test on a box without CUDA"
    return torch


def _run_worker(name, nproc, extra_env=None, args=(), timeout=300):
    """One process per GPU, torchrun-style environment, rendezvous on 127.0.0.1."""
    import socket

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    procs = []
    for r in range(nproc):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE=str(nproc), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port), PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
        env.update(extra_env or {})
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "gpu_worker.py"), name, *args],
                                      env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True))
    outs = []
    for p in procs:
        try:
            o, e = p.communicate(timeout=timeout)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append((p.returncode, o, e))
    for rc, o, e in outs:
        assert rc == 0, f"worker failed rc={rc}\nstdout:\n{o[-3000:]}\nstderr:\n{e[-3000:]}"
    return outs


# ------------------------------------------------------------------ transport executor (K1/K4/K5/K7/K8)
@pytest.mark.parametrize("env", [{}, {"BNET_PERSISTENT": "0"}, {"BNET_COPY_ENGINE": "tma"},
                                 {"BNET_NCLUSTERS": "8", "BNET_CLUSTER_SIZE": "4", "BNET_DEV_MIN_CHUNKSIZE": "4096"}],
                         ids=["persistent", "oneshot", "tma", "8x4clusters"])
def test_executor_copy_reduce_cast(env):
    _run_worker("executor", 1, extra_env=env)


def test_executor_relaunch_after_idle():
    _run_worker("executor_idle", 1, extra_env={"BNET_KERNEL_IDLE_US": "100"})


# ------------------------------------------------------------------ fused optimizer / DDP engine, single GPU
def test_fused_sgd_matches_torch_single_gpu():
    _run_worker("fused_sgd", 1)


def test_ddp_engine_trains_like_torch_sgd():
    _run_worker("ddp_engine", 1)


def test_fused_conv_blocks_match_eager():
    _run_worker("fused_nn", 1)


def test_pack_cast():
    _run_worker("pack_cast", 1)


def test_smoke_entry():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g

    g.smoke()


def test_bench_contract_single_gpu():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "3", "--warmup", "3", "--batch", "8", "--no-resnet"],
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1]
    d = json.loads(line)
    assert d["metric"] == "vgg16_train_img_per_sec" and d["n_gpus"] == 1 and d["value"] > 0
    assert d["gpu_launches"] > 0 and d["e2e"]["h2d_bytes_per_step"] > 0 and d["dtype"] == "bf16"
    ref = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference"], capture_output=True,
                         text=True, timeout=60)
    assert ref.returncode == 0 and json.loads(ref.stdout.splitlines()[-1])["impl"] == "reference"


# ------------------------------------------------------------------ multi-GPU: collectives, plugin, NCCL in the loop
@pytest.mark.multigpu
def test_allreduce_kernels_2gpu():
    _run_worker("allreduce", 2)


@pytest.mark.multigpu
def test_fused_sgd_2gpu_matches_reference():
    _run_worker("fused_sgd", 2)


@pytest.mark.multigpu
def test_ddp_engine_2gpu():
    _run_worker("ddp_engine", 2)


@pytest.mark.multigpu
def test_plugin_nvl_transport_with_cuda_buffers():
    from conftest import run_pair

    outs = run_pair(["--mem", "cuda", "--sizes", "0,1,8,4096,524288,1048577,4194304", "--inflight", "8", "--rounds", "2"],
                    env={"BNET_NVL": "1"}, timeout=240)
    for rc, res, err in outs:
        assert res is not None and rc == 0 and res["ok"], (res, err[-3000:])
        assert res["transport"] == "nvl"
    sender = outs[1][1]
    assert sender["exec"]["chunks"] > 0, f"device kernels were not used: {sender}"


@pytest.mark.multigpu
def test_nccl_loads_plugin_and_allreduces():
    from bagua_net_b200.utils.env import nccl_plugin_env

    env = nccl_plugin_env(force_net=True, debug=True)
    outs = _run_worker("nccl_allreduce", 2, extra_env=env, timeout=300)
    log = "".join(o + e for _, o, e in outs)
    assert "Using network BNet" in log or "NET/Plugin: Loaded net plugin BNet" in log, log[-4000:]


# ------------------------------------------------------------------ newest paths last (a failure here must not hide the rest under -x);
# ordered from plain Python compositions of validated kernels to new device-side modes
def test_ddp_loader_loop_and_checkpoint():
    _run_worker("ddp_api", 1, timeout=240)


@pytest.mark.multigpu
def test_ddp_loader_loop_and_checkpoint_2gpu():
    _run_worker("ddp_api", 2, timeout=240)


def test_lr_schedule_through_device_resident_hyperparameters():
    _run_worker("lr_schedule", 1, timeout=240)


@pytest.mark.multigpu
def test_collectives_on_ordinary_tensors_2gpu():
    _run_worker("collectives_any", 2, timeout=240)


def test_fused_batchnorm_blocks_match_eager():
    _run_worker("fused_bn", 1, timeout=240)


def test_executor_fp8_e5m2_ops():
    _run_worker("executor_e5m2", 1, timeout=120)


def test_executor_copy_engine_mode():
    """BNET_COPY_ENGINE=ce: plain copies ride the DMA engines + a stream-ordered completion word; the fused
    reduce/cast ops still use the cluster kernels."""
    _run_worker("executor", 1, extra_env={"BNET_COPY_ENGINE": "ce"}, timeout=120)


@pytest.mark.multigpu
def test_plugin_nvl_transport_copy_engine_mode():
    from conftest import run_pair

    outs = run_pair(["--mem", "cuda", "--sizes", "0,1,8,4096,524288,1048577,4194304", "--inflight", "8", "--rounds", "2"],
                    env={"BNET_NVL": "1", "BNET_COPY_ENGINE": "ce"}, timeout=240)
    for rc, res, err in outs:
        assert res is not None and rc == 0 and res["ok"], (res, err[-3000:])
        assert res["transport"] == "nvl"


@pytest.mark.parametrize("env", [{"BNET_EXEC_GRID": "1"}, {"BNET_EXEC_GRID": "1", "BNET_COPY_ENGINE": "tma"}], ids=["grid", "grid-tma"])
def test_executor_single_grid_mode(env):
    """BNET_EXEC_GRID=1: all cluster queues served by ONE resident grid on one stream (one launch per wake-up)."""
    _run_worker("executor", 1, extra_env=env, timeout=120)
    _run_worker("executor_idle", 1, extra_env=dict(env, BNET_KERNEL_IDLE_US="100"), timeout=60)


# ------------------------------------------------------------------ wgmma linear / convolution / fused GEMM + all-reduce
# (the kernel's waits carry a watchdog, so a wrong pipeline fails instead of hanging)
def test_tcgen05_linear_matches_fp32_reference():
    _run_worker("tc_linear", 1, timeout=240)


def test_tcgen05_conv3x3_matches_cudnn():
    _run_worker("tc_conv", 1, timeout=240)


@pytest.mark.multigpu
def test_tcgen05_row_parallel_linear_2gpu():
    _run_worker("tc_row_parallel", 2, timeout=240)


# ------------------------------------------------------------------ round 2: advisor's race, the collective on the transport
def test_fused_sgd_many_staggered_ctas_single_gpu():
    _run_worker("fused_sgd_staggered", 1, timeout=240)


@pytest.mark.multigpu
def test_fused_sgd_many_staggered_ctas_2gpu():
    _run_worker("fused_sgd_staggered", 2, timeout=240)


@pytest.mark.multigpu
def test_transport_ring_allreduce_2gpu():
    """The all-reduce that rides the transport: fused isend-reduce hops between plugin connections, on real NVLink."""
    _run_worker("transport_ring", 2, timeout=300)


@pytest.mark.multigpu
def test_transport_ring_compressed_allreduce_2gpu():
    _run_worker("transport_ring_compressed", 2)


@pytest.mark.multigpu
def test_transport_mesh_oneshot_allreduce_2gpu():
    _run_worker("transport_mesh", 2)


@pytest.mark.multigpu
def test_transport_mesh_twoshot_allreduce_2gpu():
    """Reduce-scatter by fused isend into the slice owner + all-gather by copy; in place; ranks end with identical bits."""
    _run_worker("transport_mesh_twoshot", 2)


def _run_script(script, nproc, timeout=300):
    """A benchmark script of bench/ as one process per GPU (torchrun-style environment); returns rank 0's JSON line."""
    import socket

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    procs = []
    for r in range(nproc):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE=str(nproc), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port),
                   PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "bench", script)], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.PIPE, text=True))
    outs = []
    for p in procs:
        try:
            o, e = p.communicate(timeout=timeout)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        outs.append((p.returncode, o, e))
    for rc, o, e in outs:
        assert rc == 0, f"{script} failed rc={rc}\nstdout:\n{o[-2000:]}\nstderr:\n{e[-3000:]}"
    return json.loads([ln for ln in outs[0][1].splitlines() if ln.startswith("{")][-1]), "".join(o + e for _, o, e in outs)


@pytest.mark.multigpu
def test_transport_collectives_bench_2gpu():
    """bench/transport_coll.py (what bench.py reports as extra.transport_allreduce): ring, two-shot and one-shot all-reduces
    over the plugin's own connections, exact on every rank."""
    d, _ = _run_script("transport_coll.py", 2)
    assert d["exact"] and d["transport"] == "nvl" and d["two_shot_fp32_in_place"] and d["ring_fp32"], d


@pytest.mark.multigpu
def test_nccl_collnet_probe_2gpu():
    """bench/nccl_collnet_probe.py: NCCL with the plugin's CollNet table switched on must at least produce exact all-reduces
    (whether it ran them THROUGH the table is what `collnet_allreduces_min_over_ranks` reports)."""
    d, log = _run_script("nccl_collnet_probe.py", 2)
    assert d["exact"], d
    print("collnet all-reduces executed by the plugin (min over ranks):", d["collnet_allreduces_min_over_ranks"])


# ------------------------------------------------------------------ the newest paths: LAST in the file
def test_executor_fp8_decompression_ops():
    """fp8 -> fp32 overwrite ops (OP_CAST_E4M3_TO_F32 / OP_CAST_E5M2_TO_F32) of the compressed all-reduce's all-gather half."""
    _run_worker("executor_decompress", 1, timeout=120)


def test_tcgen05_conv3x3_filter_gradient_matches_cudnn():
    """wgmma weight gradient (both operands 64-pixel 4-D TMA boxes, MN-major; split over the pixels with the fix-up)."""
    _run_worker("tc_conv_wgrad", 1, timeout=300)


def test_adopted_gradients_self_check():
    """parallel/ddp.py::direct_grads_self_check — what bench.py asks before the flagship run relies on adopted gradients."""
    _run_worker("grads_check", 1, timeout=300)

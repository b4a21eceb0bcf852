"""pytest config: registers the `gpu` marker and makes sure the native library exists.

CPU tests (`-m "not gpu"`) exercise the host engine, the TCP/shared-memory transports
and the plugin ABI over loopback; GPU tests (`-m gpu`) need a real H100.
"""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")
    config.addinivalue_line("markers", "multigpu: needs >= 2 CUDA devices")


def pytest_sessionfinish(session, exitstatus):
    # workers that are killed on purpose (peer-death tests) cannot unlink their emulated device segments
    import glob

    for f in glob.glob("/dev/shm/bnet-fake-*"):
        try:
            pid = int(os.path.basename(f).split("-")[2])
            os.kill(pid, 0)            # still alive: not ours to remove
        except (ValueError, IndexError, PermissionError):
            continue
        except ProcessLookupError:
            try:
                os.unlink(f)
            except OSError:
                pass


@pytest.fixture(scope="session", autouse=True)
def native_lib():
    import bagua_net_b200

    path = bagua_net_b200.build()
    assert os.path.exists(path)
    return path


def _gpu_count():
    try:
        import torch

        return torch.cuda.device_count() if torch.cuda.is_available() else 0
    except Exception:
        return 0


def pytest_collection_modifyitems(config, items):
    n = None
    for item in items:
        if "multigpu" in item.keywords:
            if n is None:
                n = _gpu_count()
            if n < 2:
                item.add_marker(pytest.mark.skip(reason="needs >= 2 GPUs"))


def run_pair(args, env=None, timeout=120):
    """Launch receiver (role 0) and sender (role 1) of tests/loopback_worker.py; return their JSON lines."""
    import json
    import tempfile

    worker = os.path.join(ROOT, "tests", "loopback_worker.py")
    e = dict(os.environ)
    e["PYTHONPATH"] = ROOT + os.pathsep + e.get("PYTHONPATH", "")
    e.update(env or {})
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, worker, str(role), d] + list(args), env=e,
                                  stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for role in (0, 1)]
        outs = []
        for p in procs:
            try:
                o, err = p.communicate(timeout=timeout)
            except subprocess.TimeoutExpired:
                for q in procs:
                    q.kill()
                raise
            line = [ln for ln in o.splitlines() if ln.startswith("{")]
            outs.append((p.returncode, json.loads(line[-1]) if line else None, err))
    return outs


def run_ring(world, args=(), env=None, timeout=180):
    """Launch `world` ranks of tests/ring_worker.py (ring all-reduce over the ncclNet table); return their JSON lines."""
    import json
    import tempfile

    worker = os.path.join(ROOT, "tests", "ring_worker.py")
    e = dict(os.environ)
    e["PYTHONPATH"] = ROOT + os.pathsep + e.get("PYTHONPATH", "")
    e.update(env or {})
    with tempfile.TemporaryDirectory() as d:
        procs = [subprocess.Popen([sys.executable, worker, str(r), str(world), d] + list(args), env=e,
                                  stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for r in range(world)]
        outs = []
        for p in procs:
            try:
                o, err = p.communicate(timeout=timeout)
            except subprocess.TimeoutExpired:
                for q in procs:
                    q.kill()
                raise
            line = [ln for ln in o.splitlines() if ln.startswith("{")]
            outs.append((p.returncode, json.loads(line[-1]) if line else None, err))
    return outs

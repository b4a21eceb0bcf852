#!/usr/bin/env python
"""Flagship benchmark: VGG16 bf16 data-parallel training throughput (img/s), synthetic data.

The reference's headline number is VGG16 synthetic training img/s with its plugin under NCCL
(reference README.md:52-84; BASELINE.md: 4046.6 img/s on 32 x V100 / 100 GbE).  This script
measures the same metric on N H100s of one box:

    python bench.py --gpus 1 --steps 20 --warmup 5
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
        --master-port 29500 bench.py --gpus 8 --steps 20 --warmup 5

--comm bnet (default)   our engine: flat symmetric buckets + ONE fused kernel per bucket
                        (NVLS in-switch reduce + SGD + parameter broadcast), overlapped with backward
--comm nccl-plugin      torch DDP over NCCL forced through our ncclNet plugin (BASELINE config #3/#4) — the SAME
                        fused model, captured in a CUDA graph like the default arm, so only the communication differs
--comm nccl             the same again over stock NCCL (P2P/NVLS): the comparison line for both
--impl reference        the unmodified reference: cannot be built offline (needs cargo + 191 crates)

At N > 1 the default run also measures the two DDP arms in child processes (bounded by a timeout) and reports them
under extra.nccl_plugin / extra.nccl_stock next to the headline: img/s, the all-reduce bus bandwidth 8 B - 128 MiB
over that path, and a cross-rank parameter checksum.  --no-arms skips them.  The run then repeats the arms on ResNet-50
(BASELINE config #4; extra.resnet50_bnet at any N, extra.resnet50_nccl_plugin / _nccl_stock at N > 1) as short child
jobs that only start while the run is younger than --resnet-deadline; --no-resnet skips them.  At N > 1 one more bounded
child (bench/transport_coll.py -> extra.transport_allreduce) verifies and times the all-reduces that ride the plugin's own
connections (ring, two-shot mesh, one-shot mesh; reduction fused into the isends); --no-transport-coll skips it.

Prints ONE JSON line on rank 0 (contract in the task statement).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

BASELINE_IMG_S = 4046.6   # reference README.md:68 (32 x V100, 100 GbE, with bagua-net)
_T0 = time.time()


def note(msg: str) -> None:
    """Progress on stderr (rank 0): where the wall-clock of a run goes, and where a stuck run stopped."""
    if os.environ.get("RANK", "0") == "0":
        tag = "child " if os.environ.get("BNET_BENCH_CHILD") else ""
        print(f"[bench {tag}+{time.time() - _T0:6.1f}s] {msg}", file=sys.stderr, flush=True)


# ---- the headline survives whatever the optional measurements do -------------------------------------------------------------
# Once the timed region is over, main() fills _HEADLINE.  If an optional measurement afterwards hangs (a child arm that cannot be
# killed, a collective a peer never enters) the watchdog prints the contract's JSON line from it — without the extras that were
# not finished — and ends the process with exit code 0; every rank runs the same timer, so the job ends together.
_HEADLINE: dict = {}
_CHILDREN: list = []          # Popen objects of child arms that are still running (killed by the watchdog, exact pids)
_PRINT_LOCK = threading.RLock()


def headline_line(reason: str | None = None) -> str:
    h = _HEADLINE
    a = h["args"]
    out = {"metric": f"{a.model}_train_img_per_sec", "value": round(h["img_s"], 2), "unit": "img/s", "n_gpus": h["world"],
           "steps": a.steps, "warmup": a.warmup, "ms_per_step": round(h["ms_step"], 3), "higher_is_better": True,
           "scaling": "weak", "vs_baseline": round(h["img_s"] / BASELINE_IMG_S, 4), "dtype": "bf16",
           "data": "synthetic (random images/labels, random-init weights)",
           "config": {"model": a.model, "global_batch": h["world"] * a.batch, "per_gpu_batch": a.batch, "seq_len": None,
                      "image": [3, a.image, a.image], "parallelism": f"dp{h['world']}", "comm": a.comm, "path": h["path"],
                      "fused_conv_blocks": h["fused"], "cuda_graph": h["graph_used"], "params": h["n_params"],
                      "l2": "no explicit flush: per-step working set (553 MB params+grads, activations) exceeds the 50 MB L2",
                      **({"safe_level": int(os.environ["BNET_BENCH_SAFE_LEVEL"])} if os.environ.get("BNET_BENCH_SAFE_LEVEL") else {})},
           "clocks": h["clocks"], "gpu_launches": h["nlaunch"], "wall_ms_per_step": round(h["wall_ms"], 3)}
    if h.get("checksum"):
        out["param_checksum"] = h["checksum"]
    if h.get("e2e"):
        out["e2e"] = h["e2e"]
    extra = dict(h.get("extra") or {})
    if reason:
        extra["cut_short"] = reason
    if extra:
        out["extra"] = extra
    return json.dumps(out)


def _watchdog_fire(reason: str) -> None:
    try:
        _watchdog_fire_inner(reason)
    finally:
        os._exit(0)


def _watchdog_fire_inner(reason: str) -> None:
    for proc in list(_CHILDREN):
        try:
            proc.kill()
        except Exception:   # noqa: BLE001
            pass
    with _PRINT_LOCK:
        if _HEADLINE.get("rank") == 0 and not _HEADLINE.get("printed"):
            _HEADLINE["printed"] = True
            try:
                line = headline_line(reason)
            except Exception:   # noqa: BLE001 - e.g. the main thread was adding to `extra` at this very moment
                _HEADLINE["extra"] = {}
                line = headline_line(reason)
            a = _HEADLINE["args"]
            if a.child_json:
                try:
                    with open(a.child_json + ".tmp", "w") as f:
                        f.write(line)
                    os.replace(a.child_json + ".tmp", a.child_json)
                except Exception:   # noqa: BLE001
                    pass
            print(line, flush=True)
    sys.stderr.flush()
    if _HEADLINE.get("rank") != 0:
        time.sleep(2.0)         # rank 0's line first
    os._exit(0)


def arm_watchdog() -> None:
    """Every optional part of the run is bounded (child timeouts, nothing optional starts after --resnet-deadline), so a
    complete run is over well before this fires.  BNET_BENCH_HARD_DEADLINE: seconds since start (unset / 0: derived from the
    arm timeouts, never less than four minutes after the headline)."""
    limit = float(os.environ.get("BNET_BENCH_HARD_DEADLINE", "0") or 0)
    if limit <= 0:
        a = _HEADLINE["args"]
        limit = (a.resnet_deadline + max(a.resnet_timeout, a.arm_timeout) + 60.0) if _HEADLINE["world"] > 1 or not a.no_arms else 0
        limit = max(limit, (time.time() - _T0) + 240.0)      # never less than four minutes after the headline
    t = threading.Timer(max(limit - (time.time() - _T0), 1.0),
                        lambda: _watchdog_fire(f"optional measurements still running {limit:.0f} s after start: cut short by the watchdog"))
    t.daemon = True
    t.start()
    _HEADLINE["watchdog"] = t


def reference_arm(args):
    """The reference is Rust + C++ built by `cargo build` (reference cc/Makefile:15-16); there is no
    cargo/rustc in the image, no vendored crates and no network, and it ships no setup.py/pyproject
    for pip.  Even a prebuilt copy would be ignored by NCCL 2.27/2.28, which only probe
    ncclNetPlugin_v6+ while the reference exports v4/v3 (cc/v4/nccl_net_v4.cc:210)."""
    why = "reference needs cargo+191 crates (no rustc, no network, not pip-installable); exports only ncclNet v3/v4 which NCCL 2.28 ignores"
    probe = os.path.join(ROOT, "baseline", "_ref")
    if os.path.isdir(probe) and any(f.endswith(".so") for _, _, fs in os.walk(probe) for f in fs):
        why = "baseline/_ref exists but holds no loadable ncclNet v6+ plugin"
    if os.environ.get("RANK", "0") == "0":          # (launched under torchrun for N > 1: one line, from rank 0)
        print(json.dumps({"impl": "reference", "unavailable": why}), flush=True)
    return 0


class ClockSampler:
    """nvidia-smi clocks/throttle reasons DURING the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.idx = gpu_index
        self.rows = []
        self.proc = None
        self.th = None
        self.nvml_rows = []          # (sm MHz, max MHz, reason bitmask) every ~10 ms through NVML
        self._nvml_stop = threading.Event()
        self._nvml_th = None

    def _nvml_loop(self):
        # same counters nvidia-smi prints, read in-process so that a 100 ms timed region still gets ~10 samples
        try:
            import pynvml

            pynvml.nvmlInit()
            h = pynvml.nvmlDeviceGetHandleByIndex(self.idx)
            mx = float(pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM))
            reasons_fn = getattr(pynvml, "nvmlDeviceGetCurrentClocksEventReasons", None) or \
                pynvml.nvmlDeviceGetCurrentClocksThrottleReasons
            while not self._nvml_stop.is_set():
                self.nvml_rows.append((float(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)), mx, int(reasons_fn(h))))
                self._nvml_stop.wait(0.01)
        except Exception:
            pass                      # the nvidia-smi sampler below stays authoritative

    def start(self):
        self._nvml_th = threading.Thread(target=self._nvml_loop, daemon=True)
        self._nvml_th.start()
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "200", "-i", str(self.idx)], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
        except OSError:
            self.proc = None
            return
        self.th = threading.Thread(target=self._read, daemon=True)
        self.th.start()

    def _read(self):
        for line in self.proc.stdout:
            parts = [p.strip() for p in line.split(",")]
            if len(parts) >= 8:
                self.rows.append(parts)

    NVML_REASONS = {0x8: "hw_slowdown", 0x40: "hw_thermal_slowdown", 0x20: "sw_thermal_slowdown", 0x4: "sw_power_cap",
                    0x80: "hw_power_brake_slowdown"}

    def stop(self) -> dict:
        self._nvml_stop.set()
        if self._nvml_th:
            self._nvml_th.join(timeout=2)
        if self.proc:
            smi = self._stop_smi()
        else:
            smi = {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"], "samples": 0}
        if self.nvml_rows:
            sm = [r[0] for r in self.nvml_rows]
            bits = 0
            for r in self.nvml_rows:
                bits |= r[2]
            reasons = sorted(set(smi.get("reasons") or []) | {n for b, n in self.NVML_REASONS.items() if bits & b})
            return {"sm_mhz": statistics.median(sm), "sm_max_mhz": self.nvml_rows[0][1],
                    "reasons": [r for r in reasons if r != "nvidia-smi unavailable"], "samples": len(sm),
                    "source": "nvml (10 ms period) + nvidia-smi -lms 200", "nvidia_smi_samples": smi.get("samples", 0)}
        return smi

    def _stop_smi(self) -> dict:
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except subprocess.TimeoutExpired:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        for r in self.rows:
            try:
                sm.append(float(r[1]))
                mx.append(float(r[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[4:8]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def maybe_reexec_for_plugin(args):
    """NCCL dlopen()s the net plugin by name from LD_LIBRARY_PATH at first communicator creation;
    the loader path must be in the environment before the process starts."""
    if args.comm != "nccl-plugin" or os.environ.get("BNET_BENCH_REEXEC") == "1":
        return
    from bagua_net_b200.utils.env import nccl_plugin_env

    env = dict(os.environ)
    # CUDA_MODULE_LOADING: the helper's default (EAGER) is the safe choice for an arbitrary application, at the price of
    # minutes of start-up per process with torch's kernel libraries.  This benchmark launches every kernel of its step
    # once before a collective can be in flight (warm-up steps, single-rank DDP dry run), so lazy loading is safe HERE;
    # BNET_BENCH_MODULE_LOADING=eager brings the helper's default back.
    eager = os.environ.get("BNET_BENCH_MODULE_LOADING", "lazy").lower() == "eager"
    env.update(nccl_plugin_env(force_net=True, eager_modules=eager))
    env["BNET_BENCH_REEXEC"] = "1"
    os.execve(sys.executable, [sys.executable] + sys.argv, env)


def isolated_self_check(name: str, local: int, timeout: float = 240.0):
    """Run bagua_net_b200.ops.fused_nn.<name>() on GPU `local` in a CHILD process, so that a kernel that faults there
    (a poisoned CUDA context) costs the fused layers, not the whole benchmark.
    True / False = the check's verdict (a child killed by a signal, or still running after `timeout` seconds — a hung
    kernel — counts as False);
    None = the child could not do its job for an unrelated reason (start-up error): check in-process instead."""
    root = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "LOCAL_WORLD_SIZE", "GROUP_RANK", "MASTER_ADDR", "MASTER_PORT",
              "TORCHELASTIC_RUN_ID"):
        env.pop(k, None)                        # the child is a plain single-GPU process
    code = ("import sys\n"
            "try:\n"
            "    import torch\n"
            f"    torch.cuda.set_device({int(local)})\n"
            "    from bagua_net_b200.ops import fused_nn\n"
            "except Exception:\n"
            "    sys.exit(4)\n"
            f"sys.exit(0 if fused_nn.{name}() else 3)\n")
    try:
        rc = subprocess.run([sys.executable, "-c", code], env=env, timeout=timeout, stdout=subprocess.DEVNULL,
                            stderr=subprocess.DEVNULL).returncode
    except subprocess.TimeoutExpired:           # (subprocess.run has killed the child)
        return False
    except Exception:                           # noqa: BLE001 - spawn failure
        return None
    if rc == 0:
        return True
    if rc == 3 or rc < 0:
        return False
    return None


ARM_SIZES = (8, 1 << 10, 64 << 10, 1 << 20, 16 << 20, 128 << 20)   # all-reduce message sizes of the DDP arms (bytes)


def run_child_arm(comm_name: str, args, rank: int, world: int, port_offset: int, timeout: float, model: str | None = None,
                  script: list | None = None, extra_env: dict | None = None, tag: str = ""):
    """One DDP arm (`--comm nccl-plugin` / `--comm nccl`) as a child process per rank: own CUDA context, own NCCL
    (with or without the plugin on LD_LIBRARY_PATH), own rendezvous port.  Every rank of the parent job calls this at
    the same time; rank 0 returns the child's JSON (or a status dict), the others None.  A child that outlives
    `timeout` is killed (its exact pid) — a stalled transport costs this arm, not the benchmark."""
    import tempfile

    env = dict(os.environ)
    env["MASTER_PORT"] = str(int(os.environ.get("MASTER_PORT", "29500")) + port_offset)
    env["BNET_BENCH_CHILD"] = "1"
    # the children rendezvous on their own port: the elastic agent's store (TORCHELASTIC_USE_AGENT_STORE) lives on the
    # parent job's MASTER_PORT only, so rank 0 of the child job must host the TCPStore itself
    for k in [k for k in env if k.startswith("TORCHELASTIC_")] + ["GROUP_RANK", "ROLE_RANK", "ROLE_NAME", "ROLE_WORLD_SIZE", "GROUP_WORLD_SIZE"]:
        env.pop(k, None)
    model = model or args.model
    if model == args.model:
        env["BNET_BENCH_FUSED_VERDICT"] = "0" if args.no_fused or getattr(args, "fused_failed", False) else "1"
    else:
        env.pop("BNET_BENCH_FUSED_VERDICT", None)   # another model family: the child checks its own layer kernels
        env.pop("BNET_TC_WGRAD_CHECK_SHAPES", None)  # ... and names its own layer shapes to the filter-gradient self-check
    env.pop("BNET_BENCH_REEXEC", None)
    # a child that has its headline but not yet its side measurements when the parent's patience ends prints what it has
    # (its own watchdog, a few seconds before this process would kill it)
    env["BNET_BENCH_HARD_DEADLINE"] = str(max(timeout - 8.0, 5.0))
    env.update(extra_env or {})
    log_dir = os.environ.get("BNET_BENCH_LOG_DIR") or tempfile.gettempdir()
    os.makedirs(log_dir, exist_ok=True)
    out_path = os.path.join(log_dir, f"bnet_bench_arm_{model}_{comm_name}{tag}_{os.getppid()}_{env['MASTER_PORT']}.json")
    if rank == 0 and os.path.exists(out_path):
        os.unlink(out_path)
    if script:                                   # another measurement script with the same contract: --json <file>, rank 0 writes it
        cmd = [sys.executable] + list(script) + ["--json", out_path]
    else:
        cmd = [sys.executable, os.path.abspath(__file__), "--comm", comm_name, "--gpus", str(world), "--steps", str(min(args.steps, 10)),
               "--warmup", "3", "--model", model, "--batch", str(args.batch), "--image", str(args.image), "--no-e2e",
               "--no-arms", "--child-json", out_path]
        if args.no_fused:
            cmd.append("--no-fused")
        if args.no_graph:
            cmd.append("--no-graph")
    log_path = out_path.replace(".json", f".rank{rank}.log")
    t0 = time.time()
    status = "ok"
    with open(log_path, "w") as logf:
        proc = subprocess.Popen(cmd, env=env, stdout=logf, stderr=subprocess.STDOUT)
        _CHILDREN.append(proc)
        try:
            rc = proc.wait(timeout=timeout)
            if rc != 0:
                status = f"exit code {rc}"
        except subprocess.TimeoutExpired:
            proc.kill()
            proc.wait()
            status = f"timeout after {int(timeout)} s (killed)"
        finally:
            _CHILDREN.remove(proc)
    if rank != 0:
        return None
    res = {"status": status, "wall_s": round(time.time() - t0, 1)}
    if script:
        res["log_path"] = log_path
    try:
        with open(out_path) as f:
            res.update(json.load(f))
    except Exception:                            # noqa: BLE001
        if status == "ok":
            res["status"] = "no result written"
        try:
            with open(log_path) as f:
                tail = [ln.strip() for ln in f.read().splitlines() if ln.strip() and "Warning" not in ln]
            res["log_tail"] = tail[-6:]
        except Exception:                        # noqa: BLE001
            pass
    return res


# What a failed run is repeated with (1 GPU only; a fresh process, because a faulting kernel poisons the CUDA context):
# level 1 switches off what had not run on hardware when this round's GPU budget ended (adopted gradients, the wgmma filter
# gradient), level 2 every wgmma kernel and the CUDA graph.  The JSON line says which level produced the number
# (config.safe_level); the run itself is the full benchmark either way — same model, same step, same optimizer.
SAFE_LEVELS = ({"BNET_DIRECT_GRADS": "0", "BNET_TC_WGRAD": "0"},
               {"BNET_DIRECT_GRADS": "0", "BNET_TC_WGRAD": "0", "BNET_TC": "0", "BNET_TC_CONV": "0", "BNET_BENCH_NO_GRAPH": "1"})


DUMP_PARAM_SAMPLE = 1 << 22       # float32 elements of the parameter sample: 16 MiB


def dump_outputs(out_dir: str, loss, params) -> None:
    """What a caller of the timed training step receives after its last step: the loss it returned and the parameters it
    updated (a fixed, seeded sample of them when there are more than DUMP_PARAM_SAMPLE), as float32 .npy files."""
    import numpy as np
    import torch

    os.makedirs(out_dir, exist_ok=True)
    loss = loss if torch.is_tensor(loss) else torch.tensor(loss)
    np.save(os.path.join(out_dir, "loss.npy"), loss.detach().float().reshape(1).cpu().numpy())
    flat = params.detach().reshape(-1)
    if flat.numel() > DUMP_PARAM_SAMPLE:
        gen = torch.Generator().manual_seed(0)
        idx = torch.randint(0, flat.numel(), (DUMP_PARAM_SAMPLE,), generator=gen).sort().values
        flat = flat[idx.to(flat.device)]
    np.save(os.path.join(out_dir, "params_sample.npy"), flat.float().cpu().numpy())
    note(f"outputs of the last timed step written to {out_dir}")


def main() -> int:
    try:
        return _main()
    except SystemExit:
        raise
    except BaseException as ex:   # noqa: BLE001
        import traceback

        traceback.print_exc()
        if _HEADLINE.get("img_s") is not None:            # the timed region is over: its number is printed, come what may
            _watchdog_fire(f"{type(ex).__name__}: {str(ex)[:200]}")
        level = int(os.environ.get("BNET_BENCH_SAFE_LEVEL", "0"))
        solo = os.environ.get("WORLD_SIZE", "1") == "1"
        if (solo and level < len(SAFE_LEVELS) and "reference" not in sys.argv
                and not isinstance(ex, KeyboardInterrupt) and time.time() - _T0 < 400):
            env = dict(os.environ, **SAFE_LEVELS[level])
            env["BNET_BENCH_SAFE_LEVEL"] = str(level + 1)
            env["BNET_BENCH_SAFE_REASON"] = f"{type(ex).__name__}: {str(ex)[:160]}"
            print(f"[bench] run failed ({type(ex).__name__}); repeating in a fresh process with {SAFE_LEVELS[level]}",
                  file=sys.stderr, flush=True)
            sys.stdout.flush()
            os.execve(sys.executable, [sys.executable] + sys.argv, env)
        raise


def _main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="bnet", choices=["bnet", "reference"])
    ap.add_argument("--comm", default="bnet", choices=["bnet", "nccl", "nccl-plugin"])
    ap.add_argument("--model", default="vgg16")
    ap.add_argument("--batch", type=int, default=32, help="per-GPU batch (reference benchmark script default: 32)")
    ap.add_argument("--image", type=int, default=224)
    ap.add_argument("--bucket-mb", type=float, default=64.0)
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-extra", action="store_true", help="skip the all-reduce busbw side measurement")
    ap.add_argument("--no-arms", action="store_true", help="N > 1: skip the NCCL-over-plugin / stock-NCCL DDP arms")
    ap.add_argument("--arm-timeout", type=float, default=150.0, help="seconds one DDP arm (child processes) may take")
    ap.add_argument("--no-resnet", action="store_true", help="skip the ResNet-50 side arms (BASELINE config #4)")
    ap.add_argument("--no-transport-coll", action="store_true", help="N > 1: skip the ring / two-shot all-reduces over the plugin's connections")
    ap.add_argument("--resnet-timeout", type=float, default=90.0, help="seconds one ResNet-50 arm may take")
    ap.add_argument("--resnet-deadline", type=float, default=300.0,
                    help="no ResNet-50 arm starts once the run is this many seconds old")
    ap.add_argument("--no-prefetch", action="store_true", help="e2e: per-step API instead of the prefetching loop")
    ap.add_argument("--no-graph", action="store_true", help="launch every kernel of the step individually (no CUDA graph)")
    ap.add_argument("--no-fused", action="store_true", help="eager bias/ReLU/pool instead of the fused sm_90a conv blocks")
    ap.add_argument("--force-fused", action="store_true", help="resnet: skip the fused-vs-eager timing and use the fused blocks")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps write what the last timed step computed (loss, a fixed sample of the updated "
                         "parameters) as DIR/<name>.npy")
    ap.add_argument("--child-json", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    if args.impl == "reference":
        return reference_arm(args)
    if args.warmup < 3:
        args.warmup = 3
    if os.environ.get("BNET_BENCH_NO_GRAPH") == "1":
        args.no_graph = True
    maybe_reexec_for_plugin(args)
    if os.environ.get("BNET_BENCH_CHILD") or os.environ.get("BNET_BENCH_STACKS"):
        import faulthandler

        # a child arm that is still running shortly before its parent kills it says where it is stuck
        faulthandler.dump_traceback_later(float(os.environ.get("BNET_BENCH_STACKS", "120")), exit=False, file=sys.stderr)

    import torch
    import torch.distributed as dist

    from bagua_net_b200.models import build_model
    from bagua_net_b200.parallel import BnetDDP, init_process_group_from_env

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus and rank == 0:
        print(f"[bench] note: --gpus {args.gpus} but WORLD_SIZE={world}; using WORLD_SIZE", file=sys.stderr)
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device visible; bench.py needs an H100"}), flush=True)
        return 2
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    note(f"start: comm={args.comm} model={args.model} world={world}")
    init_process_group_from_env("nccl")
    note("process group up")
    # cuDNN's algorithms by its heuristics and among the deterministic ones only: with the same arguments every run computes
    # the same numbers (benchmark mode would pick by timing, run by run)
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    torch.manual_seed(1234)

    # every arm trains the SAME model: the one built from our fused conv blocks (when they pass their self-check)
    fused = not args.no_fused and args.model.startswith(("vgg", "resnet"))
    fused_note = None
    if fused:
        # the native layer kernels are checked against the eager chain on this very GPU before they are trusted
        # with the benchmark; all ranks take the same decision
        from bagua_net_b200.ops import fused_nn

        check = fused_nn.self_check if args.model.startswith("vgg") else fused_nn.self_check_bn
        inherited = os.environ.get("BNET_BENCH_FUSED_VERDICT")     # a child arm: the parent has run the check on this GPU
        if inherited in ("0", "1"):
            verdict = inherited == "1"
        else:
            # in-process by default (about a second); BNET_BENCH_ISOLATED_CHECK=1 runs it in a child process instead, so
            # that a faulting kernel costs the fused layers and not the benchmark (+20-40 s of process start-up)
            verdict = isolated_self_check(check.__name__, local) if os.environ.get("BNET_BENCH_ISOLATED_CHECK") == "1" else None
            if verdict is None:
                verdict = check(dev)
        note(f"fused layer self-check: {verdict}")
        ok = torch.tensor([1 if verdict else 0], device=dev, dtype=torch.int32)
        if world > 1:
            dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if int(ok.item()) == 0:
            fused, fused_note = False, "fused layer kernels failed their self-check on this machine: eager layers used"
            args.fused_failed = True
            if rank == 0:
                print(f"[bench] WARNING: {fused_note}", file=sys.stderr)
    if fused:
        # settle the wgmma kernels' once-per-process verdicts (the filter gradient's runs in a child process the first
        # time on a machine) while no collective is in flight, then line the ranks up again
        from bagua_net_b200.ops import tc_conv

        # the 3x3 / stride-1 layers this run will train, at its batch size: the filter-gradient kernel's child-process
        # self-check covers exactly these shapes too (a shape-dependent fault must not be able to happen in THIS process)
        if "BNET_TC_WGRAD_CHECK_SHAPES" not in os.environ:
            s_ = args.image
            layers = ([(64, 64, s_), (64, 128, s_ // 2), (128, 128, s_ // 2), (128, 256, s_ // 4), (256, 256, s_ // 4), (256, 512, s_ // 8),
                       (512, 512, s_ // 8), (512, 512, s_ // 16)] if args.model.startswith("vgg") else
                      [(64, 64, s_ // 4), (128, 128, s_ // 8), (256, 256, s_ // 16), (512, 512, s_ // 32)])
            os.environ["BNET_TC_WGRAD_CHECK_SHAPES"] = ";".join(f"{args.batch},{ci},{co},{hw}" for ci, co, hw in layers if hw > 0)
        try:
            note(f"wgmma kernels: {tc_conv.prepare()}")
        except Exception as ex:   # noqa: BLE001 - an unsettled verdict only means cuDNN / cuBLAS are used
            note(f"wgmma kernels: verdicts could not be settled ({ex!r})")
        if world > 1:
            dist.barrier()
    if fused and args.model.startswith("resnet") and not args.force_fused:
        # The fused BatchNorm blocks are numerically checked but their speed against cuDNN's own BatchNorm kernels was never
        # measured in a whole model: time forward + backward of both variants on this GPU (no collective involved) and train
        # the faster one; every rank takes the same decision (slowest rank's times).
        def fwd_bwd_ms(flag):
            m = build_model(args.model, **({"fused": True} if flag else {})).to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
            m.train()
            xs = torch.randn(args.batch, 3, args.image, args.image, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
            ys = torch.randint(0, 1000, (args.batch,), device=dev)
            for _ in range(3):
                torch.nn.functional.cross_entropy(m(xs).float(), ys).backward()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                torch.nn.functional.cross_entropy(m(xs).float(), ys).backward()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / 5

        try:
            t = torch.tensor([fwd_bwd_ms(True), fwd_bwd_ms(False)], device=dev, dtype=torch.float64)
            if world > 1:
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
            t_fused, t_eager = float(t[0].item()), float(t[1].item())
            note(f"{args.model} forward+backward: fused blocks {t_fused:.2f} ms, eager layers {t_eager:.2f} ms")
            if t_eager < t_fused:
                fused = False
                fused_note = f"eager layers are faster on this GPU ({t_eager:.2f} ms vs {t_fused:.2f} ms forward+backward): eager layers used"
            else:
                fused_note = f"fused blocks {t_fused:.2f} ms vs eager layers {t_eager:.2f} ms forward+backward"
        except Exception as ex:   # noqa: BLE001 - the comparison is optional
            note(f"fused-vs-eager timing failed: {ex!r}")
        torch.cuda.empty_cache()
    grads_check = None
    if (args.comm == "bnet" and os.environ.get("BNET_DIRECT_GRADS", "1") != "0" and os.environ.get("BNET_BENCH_GRADS_CHECK", "1") != "0"):
        # Gradients written straight into the engine's flat buffer ("adopted", ops/grad_target.py) must train like accumulated
        # ones on THIS machine before the benchmark relies on them: two small engines, same seed, fp32 updates compared — on a
        # single-rank group (nothing in the check waits for a peer); every rank takes the same decision.  A failed check is not
        # an error: the run then accumulates (BNET_DIRECT_GRADS=0, inherited by the child arms) and says so in the JSON line.
        from bagua_net_b200.parallel.ddp import direct_grads_self_check

        solo = [dist.new_group([r]) for r in range(world)][rank] if world > 1 else None
        ok_, grads_check = direct_grads_self_check(dev, group=solo, fused=fused)
        flag = torch.tensor([1 if ok_ else 0], device=dev, dtype=torch.int32)
        if world > 1:
            dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        grads_check = dict(grads_check, passed=bool(ok_), used=bool(int(flag.item())))
        note(f"adopted-gradient self-check: {grads_check}")
        if int(flag.item()) == 0:
            os.environ["BNET_DIRECT_GRADS"] = "0"
        torch.cuda.empty_cache()
        torch.manual_seed(1234)
    model = build_model(args.model, **({"fused": True} if fused else {}))
    model = model.to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
    model.train()
    lr, mom, wd = 0.01, 0.9, 1e-4
    n_params = sum(p.numel() for p in model.parameters())
    B, S = args.batch, args.image
    x_dev = torch.randn(B, 3, S, S, device=dev, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y_dev = torch.randint(0, 1000, (B,), device=dev)
    graph_used = False
    graph_note = None

    def our_launches():
        from bagua_net_b200.ops import fused_nn, tc_linear

        return fused_nn.LAUNCHES + tc_linear.LAUNCHES

    if args.comm == "bnet":
        engine = BnetDDP(model, lr=lr, momentum=mom, weight_decay=wd, bucket_mb=args.bucket_mb,
                         extra_heap_bytes=384 << 20)
        comm = engine.comm
        if not args.no_graph:
            engine.enable_cuda_graph(True)
            graph_used = True

        def step_dev(x, y):
            return engine.train_step(x, y)

        def step_host(xh, yh):
            return engine.train_step_from_host(xh, yh)

        def loop_host(xh, yh, steps):
            # the loader-facing API: one H2D copy per step (prefetched under the previous step) and one
            # loss read per step; exactly `steps` batches are copied, all of them inside the timed region
            n = 0
            for _ in engine.train_from_host((xh, yh) for _ in range(steps)):
                n += 1
            assert n == steps

        def launches():
            return comm.launches + our_launches()

        def param_vector():
            return engine.flat_param
        path = ("nvls" if (comm.has_multicast and world > 2) else "p2p") if world > 1 else "single"
    else:
        # ---- torch DDP over NCCL (stock, or forced through the bnet plugin) ----------------------------------------
        # Let cuDNN pick its algorithms (and torch's allocator settle) BEFORE any collective is in flight: the
        # autotuner's emptyCache() -> cudaFree waits for the device, and a collective that is waiting for a peer which
        # is itself stuck behind such a call is the classic NCCL dead-lock (NCCL documents it for its own kernels).
        # The same goes for CUDA's lazy module loading (first launch of a kernel = a wait for the device): every kernel of a
        # training step — optimizer included — is launched once HERE, with no collective in flight, and the plugin arm
        # additionally runs with CUDA_MODULE_LOADING=EAGER (bagua_net_b200/utils/env.py explains the dead-lock).
        opt = torch.optim.SGD(model.parameters(), lr=lr, momentum=mom, weight_decay=wd)
        state0 = [p.detach().clone() for p in model.parameters()]
        for _ in range(2):
            opt.zero_grad(set_to_none=True)
            torch.nn.functional.cross_entropy(model(x_dev).float(), y_dev).backward()
            opt.step()
        with torch.no_grad():                          # (the warm-up steps must not count as training)
            for p_, s_ in zip(model.parameters(), state0):
                p_.copy_(s_)
        opt = torch.optim.SGD(model.parameters(), lr=lr, momentum=mom, weight_decay=wd)
        del state0
        model.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        if world > 1:
            # DDP's OWN kernels (bucket copies, the 1/world scaling, the bucket rebuild after the first iteration) get their
            # first launch here, through a process group of this rank alone: its collectives never wait for a peer, so a
            # module load that synchronises the context has nothing to dead-lock with.  (new_group is collective: every
            # rank creates every group.)  No optimizer step, the gradients are dropped afterwards.
            solo = [dist.new_group([r]) for r in range(world)][rank]
            with torch.cuda.stream(side):
                dry = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local], process_group=solo,
                                                                gradient_as_bucket_view=True)
                for _ in range(3):
                    torch.nn.functional.cross_entropy(dry(x_dev).float(), y_dev).backward()
                t_ = torch.ones(1024, device=dev, dtype=torch.bfloat16)
                t_.div_(float(world)).mul_(1.0 / world)
                torch.cat([t_, t_]).float().sum().item()
            del dry, t_
            model.zero_grad(set_to_none=True)
            torch.cuda.synchronize()
            note("DDP dry run on a single-rank group done")
        with torch.cuda.stream(side):                # DDP built (and warmed up) on a side stream: required for capture
            ddp = (torch.nn.parallel.DistributedDataParallel(model, device_ids=[local], gradient_as_bucket_view=True)
                   if world > 1 else model)
            gx, gy = x_dev.clone(), y_dev.clone()

            def eager_step(x, y):
                opt.zero_grad(set_to_none=True)
                loss = torch.nn.functional.cross_entropy(ddp(x).float(), y)
                loss.backward()
                opt.step()
                return loss.detach()

            note("DDP built; eager iterations")
            for _ in range(4 if world == 1 else 11):  # (DDP wants 11 eager iterations before a capture)
                eager_step(gx, gy)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        note("eager iterations done")
        graph = None
        if not args.no_graph:
            try:
                l0 = our_launches()
                opt.zero_grad(set_to_none=True)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    gloss = torch.nn.functional.cross_entropy(ddp(gx).float(), gy)
                    gloss.backward()
                    opt.step()
                graph_launches = our_launches() - l0
                graph.replay()
                torch.cuda.synchronize()
                graph_used = True
            except Exception as ex:               # noqa: BLE001 - keep the arm alive without the graph
                graph = None
                graph_note = f"capture failed ({type(ex).__name__}: {str(ex)[:120]}): eager launches"
                torch.cuda.synchronize()
        ok = torch.tensor([1 if graph is not None else 0], device=dev, dtype=torch.int32)
        if world > 1:
            dist.all_reduce(ok, op=dist.ReduceOp.MIN)     # every rank replays, or none does
        if int(ok.item()) == 0:
            graph, graph_used = None, False

        def step_dev(x, y):
            if graph is None:
                return eager_step(x, y)
            from bagua_net_b200.ops import fused_nn

            gx.copy_(x, non_blocking=True)
            gy.copy_(y, non_blocking=True)
            graph.replay()
            fused_nn.LAUNCHES += graph_launches
            return gloss

        def step_host(xh, yh):
            x = xh.to(dev, non_blocking=True).contiguous(memory_format=torch.channels_last)
            y = yh.to(dev, non_blocking=True)
            return float(step_dev(x, y).item())

        def launches():
            return our_launches()

        def param_vector():
            return torch.cat([p.detach().reshape(-1).float() for p in model.parameters()])
        comm = None
        path = args.comm

    # pinned, already in the layout the model consumes (NHWC): the H2D copy is one plain DMA
    x_host = torch.randn(B, 3, S, S, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last).pin_memory()
    y_host = torch.randint(0, 1000, (B,)).pin_memory()

    def sync_all():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps, whole=False):
        sync_all()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        if whole:
            fn(steps)            # fn runs all `steps` steps itself
        else:
            for _ in range(steps):
                fn()
        e1.record()
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3
        ms = e0.elapsed_time(e1)
        t = torch.tensor([ms, wall], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)     # max over ranks
        sync_all()
        return float(t[0].item()), float(t[1].item())

    # ---- device-resident inputs (the synthetic benchmark the reference quotes) ----------------
    note(f"engine ready (cuda graph: {graph_used}{', ' + graph_note if graph_note else ''}); warm-up")
    for _ in range(args.warmup):
        step_dev(x_dev, y_dev)
    torch.cuda.synchronize()
    note("timed region")
    sampler = ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()
    l0 = launches()
    last = {}
    ms_total, wall_total = timed(lambda: last.__setitem__("loss", step_dev(x_dev, y_dev)), args.steps)
    nlaunch = launches() - l0
    clocks = sampler.stop() if sampler else None
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last["loss"], param_vector())
    ms_step = ms_total / args.steps
    img_s = world * B / (ms_step / 1e3)

    note(f"timed: {ms_step:.3f} ms/step")
    # ---- from here on the headline exists: nothing that follows may lose it.  `headline` is what a watchdog (below) or the
    #      exception handler around the optional measurements prints if the rest of the run does not get to its end.
    checksum, e2e, extra, arms = None, None, {}, {}
    _HEADLINE.update({"extra": extra, "args": args, "world": world, "rank": rank, "img_s": img_s, "ms_step": ms_step, "clocks": clocks,
                      "nlaunch": nlaunch, "wall_ms": wall_total / args.steps, "path": path, "fused": fused,
                      "graph_used": graph_used, "n_params": n_params})
    arm_watchdog()
    try:
        # ---- cross-rank numerics: after the timed steps every rank must hold the same parameters ----
        pv = param_vector()
        csum = torch.stack([pv.double().sum(), pv.double().abs().sum()])
        checksum = {"sum": float(csum[0].item()), "abs_sum": float(csum[1].item()), "finite": bool(torch.isfinite(csum).all().item())}
        if world > 1:
            allc = [torch.zeros_like(csum) for _ in range(world)]
            dist.all_gather(allc, csum)
            torch.cuda.synchronize()      # (no first-time kernel launch while a collective is in flight: lazy module loading)
            checksum["ranks_agree"] = all(bool(torch.equal(allc[0], c)) for c in allc)
        _HEADLINE["checksum"] = checksum
        del pv

        # ---- end to end through the public API: pinned-host batch in, loss value out, every step ----
        if not args.no_e2e:
            for _ in range(args.warmup):
                step_host(x_host, y_host)
            api = "train_step_from_host"
            ms_e2e = None
            if args.comm == "bnet" and not args.no_prefetch:
                try:
                    loop_host(x_host, y_host, args.warmup)
                    ms_e2e, _ = timed(lambda k: loop_host(x_host, y_host, k), args.steps, whole=True)
                    api = "train_from_host (next batch's H2D copy prefetched under the running step)"
                except Exception as ex:     # keep the plain per-step path as the end-to-end number
                    print(f"[bench] prefetching loop failed ({ex!r}); timing train_step_from_host", file=sys.stderr)
                    ms_e2e = None
            if ms_e2e is None:
                ms_e2e, _ = timed(lambda: step_host(x_host, y_host), args.steps)
            e2e = {"value": world * B / (ms_e2e / args.steps / 1e3), "unit": "img/s",
                   "h2d_bytes_per_step": x_host.numel() * x_host.element_size() + y_host.numel() * y_host.element_size(),
                   "d2h_bytes_per_step": 4, "ms_per_step": ms_e2e / args.steps, "api": api}
            _HEADLINE["e2e"] = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in e2e.items()}

        # ---- side measurement: all-reduce bus bandwidth (BASELINE.json configs #2 / #5) ----
        if args.comm == "bnet" and world > 1 and not args.no_extra:
            try:
                bw, lat, blocks_tried = {}, {}, {}
                for nbytes in (1 << 10, 64 << 10, 1 << 20, 16 << 20, 128 << 20):     # BASELINE config #5 (1 KiB .. 128 MiB here)
                    t = comm.alloc(nbytes // 2, torch.bfloat16)
                    t.fill_(1.0)
                    for _ in range(5):
                        comm.all_reduce(t, "sum")
                    iters = 50 if nbytes <= (1 << 20) else 20
                    ms, _ = timed(lambda: comm.all_reduce(t, "sum"), iters)
                    if nbytes >= (16 << 20):
                        # The CTA count of the bandwidth kernels was tuned on 2 GPUs (32 for the in-switch path); what is best
                        # with this many ranks is measured here, on this box: same kernel, same check (max over ranks), the
                        # fastest count is reported together with the default's time.
                        tried = {"default": round(ms / iters * 1e3, 1)}
                        for nb in (48, 64, 96, 132):
                            for _ in range(3):
                                comm.all_reduce(t, "sum", nblocks=nb)
                            ms_nb, _ = timed(lambda: comm.all_reduce(t, "sum", nblocks=nb), iters)
                            tried[str(nb)] = round(ms_nb / iters * 1e3, 1)
                            if ms_nb < ms:
                                ms = ms_nb
                        blocks_tried[str(nbytes)] = tried
                    algbw = nbytes / (ms / iters / 1e3) / 1e9
                    bw[str(nbytes)] = round(algbw * 2 * (world - 1) / world, 2 if nbytes < (1 << 20) else 1)
                    lat[str(nbytes)] = round(ms / iters * 1e3, 1)
                extra["allreduce_busbw_gbs_bf16"] = bw
                extra["allreduce_time_us"] = lat
                if blocks_tried:
                    extra["allreduce_time_us_by_cta_count"] = blocks_tried
                # bytes per direction per GPU: in-switch path S(1+1/n), direct two-shot S(n-1)/n
                per_dir = (1 + 1 / world) if path == "nvls" else (world - 1) / world
                extra["allreduce_algo"] = path
                # against the nominal NVLink 4 bandwidth of an H100 SXM, 450 GB/s per direction (data sheet, not a measured peak)
                extra["allreduce_roofline_frac_of_450GBs"] = {k: round(v / (2 * (world - 1) / world) * per_dir / 450.0, 3)
                                                              for k, v in bw.items() if int(k) >= (1 << 20)}
            except Exception as ex:   # the headline number must survive a failing side measurement
                extra["allreduce_error"] = str(ex)[:200]
        if args.comm != "bnet" and world > 1 and not args.no_extra:
            # the nccl-tests sweep of the reference's README (all_reduce_perf -b 8 -e 128M), through torch.distributed:
            # bf16 sum, device-timed, max over ranks; busbw = algbw * 2(n-1)/n
            try:
                bw, lat = {}, {}
                for nbytes in ARM_SIZES:
                    t = torch.ones(max(nbytes // 2, 1), device=dev, dtype=torch.bfloat16)
                    iters = 20 if nbytes <= (16 << 20) else 8
                    for _ in range(3):
                        dist.all_reduce(t)
                    ms, _ = timed(lambda: dist.all_reduce(t), iters)
                    us = ms / iters * 1e3
                    lat[str(nbytes)] = round(us, 1)
                    bw[str(nbytes)] = round(nbytes / (us * 1e-6) / 1e9 * 2 * (world - 1) / world, 2)
                    del t
                extra["allreduce_busbw_gbs_bf16"] = bw
                extra["allreduce_time_us"] = lat
                # numerics of the path itself: sum of rank-patterned data against the closed form
                t = torch.full((1 << 20,), float(rank + 1), device=dev, dtype=torch.float32)
                torch.cuda.synchronize()
                dist.all_reduce(t)
                torch.cuda.synchronize()
                extra["allreduce_exact"] = bool((t == float(world * (world + 1) // 2)).all().item())
            except Exception as ex:   # noqa: BLE001
                extra["allreduce_error"] = str(ex)[:200]

        # ---- N > 1: the DDP arms over NCCL (through the plugin / stock) in child processes ----
        if args.comm == "bnet" and world > 1 and not args.no_arms and not os.environ.get("BNET_BENCH_CHILD"):
            sync_all()
            for i, (key, comm_name) in enumerate((("nccl_plugin", "nccl-plugin"), ("nccl_stock", "nccl"))):
                # (BNET_BENCH_MODULE_LOADING=eager: every process of the plugin arm loads all of torch's kernels up front,
                # 100 s at 2 ranks and 260 s at 4 — see maybe_reexec_for_plugin)
                slow = comm_name == "nccl-plugin" and os.environ.get("BNET_BENCH_MODULE_LOADING", "lazy").lower() == "eager"
                tmo = args.arm_timeout * (3.0 if slow else 1.0)
                note(f"arm {comm_name}: child processes (timeout {tmo:.0f} s)")
                res = run_child_arm(comm_name, args, rank, world, 101 + 37 * i, tmo)
                note(f"arm {comm_name}: {res.get('status') if res else None}")
                if world > 1:
                    dist.barrier()
                if rank == 0:
                    arms[key] = res

        # ---- the collectives that ride the transport (ring / two-shot / one-shot over the plugin's own connections, reduction
        #      fused into the isends; bench/transport_coll.py) as a bounded child job: verified exact, host-timed, max over ranks
        if (args.comm == "bnet" and world > 1 and not args.no_arms and not args.no_transport_coll and not os.environ.get("BNET_BENCH_CHILD")):
            sync_all()
            go = torch.tensor([1 if time.time() - _T0 < args.resnet_deadline else 0], device=dev, dtype=torch.int32)
            dist.broadcast(go, 0)
            if int(go.item()):
                note("transport collectives: child processes (timeout 75 s)")
                res = run_child_arm("transport", args, rank, world, 150, 75.0, model="coll",
                                    script=[os.path.join(ROOT, "bench", "transport_coll.py")])
                note(f"transport collectives: {res.get('status') if res else None}")
                dist.barrier()
                if rank == 0 and res is not None:
                    extra["transport_allreduce"] = {k: v for k, v in res.items() if k not in ("note", "log_path")}

        # ---- N = 1: where does the step go?  (tools/step_profile.py in a child: torch.profiler over eager steps of the same model;
        #      kernel names, launches and time per step — explains the number above, is not a bench value)
        if (args.comm == "bnet" and world == 1 and args.model == "vgg16" and not args.no_arms and not args.no_resnet
                and not os.environ.get("BNET_BENCH_CHILD")):
            note("step profile: child process (timeout 90 s)")
            res = run_child_arm("profile", args, rank, world, 140, 90.0, tag="_step",      # (same model: the kernels' verdicts are cached)
                                script=[os.path.join(ROOT, "tools", "step_profile.py"), "--fused", "--batch", str(args.batch), "--steps", "4"])
            note(f"step profile: {res.get('status') if res else None}")
            if res is not None:
                res.pop("log_path", None)
                extra["step_profile"] = res

        # ---- BASELINE config #4: the same three arms on ResNet-50 (child processes, short, under an overall deadline) ----
        # The headline stays VGG16 (the model the reference quotes its speed-up on); the reference's README benchmarks
        # ResNet-50 the same way (reference README.md:52-84), so the run reports it next to the headline while the GPUs are here.
        if (args.comm == "bnet" and args.model == "vgg16" and not args.no_arms and not args.no_resnet
                and not os.environ.get("BNET_BENCH_CHILD")):
            sync_all()
            # (order = what is kept if the deadline cuts the list short: config #4 itself first, then our engine, then the comparator)
            second = ([("resnet50_nccl_plugin", "nccl-plugin")] if world > 1 else []) + [("resnet50_bnet", "bnet")] + \
                     ([("resnet50_nccl_stock", "nccl")] if world > 1 else [])
            for i, (key, comm_name) in enumerate(second):
                # every rank takes rank 0's decision: an arm starts only while the whole run is younger than the deadline
                go = torch.tensor([1 if time.time() - _T0 < args.resnet_deadline else 0], device=dev, dtype=torch.int32)
                if world > 1:
                    dist.broadcast(go, 0)
                if int(go.item()) == 0:
                    if rank == 0:
                        arms[key] = {"status": f"skipped: the run was already {time.time() - _T0:.0f} s old (deadline {args.resnet_deadline:.0f} s)"}
                    continue
                note(f"arm resnet50/{comm_name}: child processes (timeout {args.resnet_timeout:.0f} s)")
                res = run_child_arm(comm_name, args, rank, world, 175 + 37 * i, args.resnet_timeout, model="resnet50")
                note(f"arm resnet50/{comm_name}: {res.get('status') if res else None}")
                if world > 1:
                    dist.barrier()
                if rank == 0:
                    arms[key] = res

        # ---- the reference-equivalent data path on THIS box: torch DDP over NCCL over the plugin restricted to what bagua-net does
        #      (host pointers only: NCCL stages through host memory; multi-stream TCP, here over the loopback interface; no NVLink or
        #      shared-memory transport).  The reference itself cannot be built here (--impl reference says why); this is its product
        #      re-implemented, same model, same step, so the ratio to the headline is the same-box speed-up over "what the
        #      reference gives on an 8 x H100 node".
        if (args.comm == "bnet" and world > 1 and not args.no_arms and not args.no_resnet and not os.environ.get("BNET_BENCH_CHILD")):
            sync_all()
            go = torch.tensor([1 if time.time() - _T0 < args.resnet_deadline else 0], device=dev, dtype=torch.int32)
            dist.broadcast(go, 0)
            if int(go.item()):
                note(f"arm nccl-plugin, host pointers over TCP (reference-equivalent): child processes (timeout {args.resnet_timeout:.0f} s)")
                res = run_child_arm("nccl-plugin", args, rank, world, 327, args.resnet_timeout,
                                    extra_env={"BNET_NVL": "0", "BNET_GDR": "0"}, tag="_tcp")
                note(f"arm nccl-plugin, host pointers over TCP: {res.get('status') if res else None}")
                dist.barrier()
                if rank == 0:
                    if res is not None:
                        res["note"] = ("reference-equivalent path: NCCL over the plugin with host pointers only and multi-stream TCP "
                                       "over loopback (BNET_NVL=0 BNET_GDR=0), what bagua-net does on one node")
                    arms["nccl_plugin_tcp_host_pointers"] = res

        # ---- does NCCL accept the plugin's CollNet table?  (bench/nccl_collnet_probe.py: plugin + BNET_COLLNET=1 NCCL_COLLNET_ENABLE=1,
        #      one virtual host per rank; fp32 all-reduce sweep, exactness, the plugin's own count of all-reduces it executed)
        if (args.comm == "bnet" and world > 1 and not args.no_arms and not args.no_transport_coll and not os.environ.get("BNET_BENCH_CHILD")):
            sync_all()
            go = torch.tensor([1 if time.time() - _T0 < args.resnet_deadline else 0], device=dev, dtype=torch.int32)
            dist.broadcast(go, 0)
            if int(go.item()):
                note("NCCL CollNet probe: child processes (timeout 75 s)")
                res = run_child_arm("collnet", args, rank, world, 163, 75.0, model="probe",
                                    script=[os.path.join(ROOT, "bench", "nccl_collnet_probe.py")])
                note(f"NCCL CollNet probe: {res.get('status') if res else None}")
                dist.barrier()
                if rank == 0 and res is not None:
                    try:      # what NCCL itself said about CollNet (rank 0's INFO log of the child)
                        logp = [p_ for p_ in (res.get("log_path"),) if p_]
                        lines = []
                        for lp in logp:
                            with open(lp, errors="replace") as f:
                                for ln in f:
                                    if "ollnet" in ln.lower() or "coll net" in ln.lower():
                                        ln = ln.strip().split("NCCL INFO ")[-1][:160]
                                        if ln not in lines:
                                            lines.append(ln)
                        res["nccl_log_collnet_lines"] = lines[:8]
                    except Exception:   # noqa: BLE001
                        pass
                    res.pop("log_path", None)
                    extra["nccl_collnet"] = res

        # ---- last and least: the DDP-over-plugin arm once more with the copy engines moving the bytes (BNET_EXEC_MODE=ce: no SM
        #      is taken from the backward pass; slower in isolation, never measured under overlap) — only if time is left
        if (args.comm == "bnet" and world > 1 and not args.no_arms and not args.no_resnet and not os.environ.get("BNET_BENCH_CHILD")):
            sync_all()
            go = torch.tensor([1 if time.time() - _T0 < args.resnet_deadline else 0], device=dev, dtype=torch.int32)
            dist.broadcast(go, 0)
            if int(go.item()):
                note(f"arm nccl-plugin with copy engines: child processes (timeout {args.resnet_timeout:.0f} s)")
                res = run_child_arm("nccl-plugin", args, rank, world, 290, args.resnet_timeout, extra_env={"BNET_EXEC_MODE": "ce"}, tag="_ce")
                note(f"arm nccl-plugin with copy engines: {res.get('status') if res else None}")
                dist.barrier()
                if rank == 0:
                    arms["nccl_plugin_copy_engines"] = res

    except Exception as ex:   # noqa: BLE001 - an optional measurement failed: the headline above is still printed
        import traceback

        traceback.print_exc()
        extra["post_headline_error"] = f"{type(ex).__name__}: {str(ex)[:200]}"
        if world > 1:
            # the other ranks may be waiting in a collective this rank will never enter: print what there is and leave together
            # (the watchdog does exactly that, for every rank)
            _watchdog_fire(f"rank {rank}: {extra['post_headline_error']}")

    if rank == 0:
        opt_desc = (f"sgd(lr={lr},momentum={mom},wd={wd}) fused into the collective" if args.comm == "bnet"
                    else f"torch.optim.SGD(lr={lr},momentum={mom},wd={wd})")
        out = {
            "metric": f"{args.model}_train_img_per_sec", "value": round(img_s, 2), "unit": "img/s",
            "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": round(ms_step, 3),
            "higher_is_better": True, "scaling": "weak", "vs_baseline": round(img_s / BASELINE_IMG_S, 4),
            "dtype": "bf16", "data": "synthetic (random images/labels, random-init weights)",
            "config": {"model": args.model, "global_batch": world * B, "per_gpu_batch": B, "seq_len": None,
                       "image": [3, S, S], "parallelism": f"dp{world}", "comm": args.comm, "path": path,
                       "fused_conv_blocks": fused, **({"fused_note": fused_note} if fused_note else {}),
                       "cuda_graph": graph_used, **({"graph_note": graph_note} if graph_note else {}),
                       "optimizer": opt_desc, "params": n_params, "bucket_mb": args.bucket_mb,
                       **({"safe_level": int(os.environ["BNET_BENCH_SAFE_LEVEL"]),
                           "safe_reason": os.environ.get("BNET_BENCH_SAFE_REASON")} if os.environ.get("BNET_BENCH_SAFE_LEVEL") else {}),
                       "l2": "no explicit flush: per-step working set (553 MB params+grads, activations) exceeds the 50 MB L2",
                       "baseline": "4046.6 img/s on 32xV100/100GbE (reference README.md:68)"},
            "clocks": clocks, "gpu_launches": nlaunch, "wall_ms_per_step": round(wall_total / args.steps, 3),
            "param_checksum": checksum,
        }
        if args.comm == "bnet":
            # how the gradients reached the flat buffer the fused kernels read: adopted in place (written there by their
            # producer) or copied in by the hook; counted over the eager / captured passes (graph replays repeat the captured one)
            try:
                npar = sum(1 for p_ in model.parameters() if p_.requires_grad)
                out["config"]["gradient_path"] = {"mode": "adopt" if getattr(engine, "_direct_grads", False) else "accumulate",
                                                  "parameters": npar, "copies_in_eager_and_captured_passes": int(engine.grad_copies)}
                if grads_check is not None:
                    out["config"]["gradient_path"]["self_check"] = {k: (round(v, 6) if isinstance(v, float) else v) for k, v in grads_check.items()}
            except Exception:   # noqa: BLE001 - reporting only
                pass
        try:
            # what the per-shape autotuner measured on THIS GPU (wgmma kernel vs cuDNN, us) and which one the step runs
            from bagua_net_b200.ops import tc_conv

            if tc_conv.TIMINGS or tc_conv._choice:
                out["config"]["tc_conv_autotune"] = {
                    f"{k[0]} n{k[1]} {k[2]}x{k[3]} {k[4]}->{k[5]}": dict(tc_conv.TIMINGS.get(k, {}), choice=v)
                    for k, v in sorted(tc_conv._choice.items(), key=lambda kv: str(kv[0])) if k[1] == args.batch}   # (not the self-check's shapes)
        except Exception:   # noqa: BLE001 - reporting only
            pass
        if e2e:
            out["e2e"] = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in e2e.items()}
        for key, res in arms.items():
            if res is None:
                continue
            # keep the arm compact: its headline, its sweep, its checks
            keep = {k: res.get(k) for k in ("status", "wall_s", "value", "ms_per_step", "log_tail", "note") if res.get(k) is not None}
            cfg = res.get("config") or {}
            keep.update({k: cfg.get(k) for k in ("model", "comm", "path", "cuda_graph", "fused_conv_blocks", "fused_note", "graph_note")
                         if cfg.get(k) is not None})
            if key == "resnet50_bnet" and cfg.get("tc_conv_autotune"):       # (the other arms run the headline's layer shapes)
                keep["tc_conv_autotune"] = cfg["tc_conv_autotune"]
            ex = res.get("extra") or {}
            keep.update({k: ex[k] for k in ("allreduce_busbw_gbs_bf16", "allreduce_time_us", "allreduce_exact", "allreduce_error",
                                            "cut_short", "post_headline_error") if k in ex})
            if res.get("param_checksum"):
                keep["param_checksum"] = res["param_checksum"]
            extra[key] = keep
        if extra:
            out["extra"] = extra
        line = json.dumps(out)
        with _PRINT_LOCK:
            if not _HEADLINE.get("printed"):
                _HEADLINE["printed"] = True
                if args.child_json:
                    with open(args.child_json + ".tmp", "w") as f:
                        f.write(line)
                    os.replace(args.child_json + ".tmp", args.child_json)
                print(line, flush=True)
    if world > 1:
        dist.barrier()
        if args.comm != "bnet":
            # A CUDA graph that captured NCCL collectives keeps the communicator busy: ncclCommDestroy then waits for it
            # (measured: the arm printed its result after 14 s and sat in destroy_process_group until it was killed).
            # Drop the graph first, and never let teardown outlive the measurement by more than a few seconds.
            import gc
            import threading

            threading.Timer(8.0, lambda: os._exit(0)).start()
            graph = gloss = None            # noqa: F841
            gc.collect()
            torch.cuda.synchronize()
        dist.destroy_process_group()
        if args.comm != "bnet":
            sys.stdout.flush()
            sys.stderr.flush()
            os._exit(0)
    return 0


if __name__ == "__main__":
    sys.exit(main())

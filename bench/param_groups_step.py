#!/usr/bin/env python
"""What parameter groups cost in the fused data-parallel step, on one GPU.

1. Optimizer time at the real tensor shapes of VGG16 (32 tensors, 138.4 M parameters) and ResNet-50 (161 tensors,
   25.6 M), built on the meta device and laid out in 64 MB buckets of bf16 parameters as BnetDDP lays them out, for SGD
   and AdamW:
   * fused: the ungrouped one-kernel step per bucket;
   * groups2: the grouped one-kernel step with the usual two groups (p.dim() <= 1 without weight decay, the rest with);
   * groups20: the grouped step with 10 lr-scale groups (consecutive tenths of the tensors) x decay / no decay;
   * torch_foreach / torch_fused: torch.optim.SGD / AdamW with the two groups on fp32 master tensors of the same shapes
     (foreach=True / fused=True), then the cast back to bf16.
   CUDA events time `--steps` whole steps after `--warmup`; the variants alternate for `--rounds` rounds (median).  The
   grouped kernels read and write the bytes the ungrouped ones do: SGD 20 bytes per bf16 parameter (gradient read 2,
   master and momentum read and written 16, parameter written 2; the gradient zeroing adds 2), AdamW 28.
2. End to end: BnetDDP.train_step img/s on ResNet-50, bf16, batch `--batch`, 224 x 224, under a CUDA graph, SGD without
   and with no_weight_decay_groups(model), alternating for `--e2e-rounds` rounds.

  python bench/param_groups_step.py --out profiles/param_groups_step
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))      # (`bench` is also bench.py at the root)
from lars_step import shapes, timed  # noqa: E402
from optimizer_step import DATASHEET_HBM_BPS, card  # noqa: E402
from bagua_net_b200.models import build_model  # noqa: E402
from bagua_net_b200.parallel import SymmComm  # noqa: E402
from bagua_net_b200.parallel.ddp import group_segments, plan_buckets  # noqa: E402

BYTES_PER_PARAM = {"sgd": 22, "adamw": 30}          # (with the gradient zeroing)
LR, MU, WD = 0.1, 0.9, 5e-5


def optimizer_times(args, results):
    for model in ("vgg16", "resnet50"):
        shp = shapes(model)
        numels = [int(torch.Size(s).numel()) for s in shp]
        T = len(shp)
        plan, total = plan_buckets(numels, 2, 1, 64.0)
        comm = SymmComm(2 * total * 2 + (64 << 20))
        flat_p, flat_g = comm.alloc(total, torch.bfloat16), comm.alloc(total, torch.bfloat16)
        flat_p.normal_(0, 0.02)
        flat_g.zero_()
        views = [(flat_g[s:s + n], flat_p[s:s + n]) for s, n, _ in plan]
        two = [int(len(s) <= 1) for s in shp]
        twenty = [2 * (i * 10 // T) + int(len(s) <= 1) for i, s in enumerate(shp)]
        tables = {}
        for name, group_of in (("groups2", two), ("groups20", twenty)):
            G = max(group_of) + 1
            segs = [comm.group_segments(group_segments(m, numels, group_of, s, n, 2, 1, 0), n // 8, G) for s, n, m in plan]
            rows = [[LR * (1.0 + 0.1 * (g // 2)), 0.0 if g % 2 else WD, 0.0, 0.0] for g in range(G)]
            tables[name] = (torch.tensor(rows, device="cuda"), segs)
        row = {"tensors": T, "params": sum(numels), "buckets": len(plan),
               "segments": {k: sum(s.shape[0] for s in v[1]) for k, v in tables.items()}}
        for optimizer in ("sgd", "adamw"):
            S = 2 if optimizer == "sgd" else 3
            state = [[p.float()] + [torch.zeros(p.numel(), device="cuda") for _ in range(S - 1)] for _, p in views]
            hp = torch.tensor([LR, MU, WD, 1.0] if optimizer == "sgd" else [LR, 0.9, 0.999, 1e-8, WD, 1.0, 0.0, 0.0], device="cuda")
            tparams = [torch.nn.Parameter(torch.randn(s, device="cuda") * 0.02) for s in shp]
            for t in tparams:
                t.grad = torch.randn_like(t) * 1e-3
            tgroups = [{"params": [t for t, g in zip(tparams, two) if g], "weight_decay": 0.0},
                       {"params": [t for t, g in zip(tparams, two) if not g], "weight_decay": WD}]
            cls = torch.optim.SGD if optimizer == "sgd" else torch.optim.AdamW
            kw = {"momentum": MU} if optimizer == "sgd" else {}
            opts = {k: cls(tgroups, lr=LR, **kw, **{k: True}) for k in ("foreach", "fused")}
            bf16 = [torch.empty(s, device="cuda", dtype=torch.bfloat16) for s in shp]

            def fused():
                step = comm.fused_allreduce_sgd if optimizer == "sgd" else comm.fused_allreduce_adamw
                for (g, p), st in zip(views, state):
                    if optimizer == "sgd":
                        step(g, p, *st, 0.0, 0.0, 0.0, 1.0, hp=hp)
                    else:
                        step(g, p, *st, hp)

            def grouped(name):
                groups, segs = tables[name]
                step = comm.fused_allreduce_sgd_groups if optimizer == "sgd" else comm.fused_allreduce_adamw_groups

                def run():
                    for (g, p), st, sg in zip(views, state, segs):
                        step(g, p, *st, hp, groups, sg)
                return run

            def torch_step(k):
                def run():
                    opts[k].step()
                    torch._foreach_copy_(bf16, [p.detach() for p in tparams])
                return run

            variants = {"fused": fused, "groups2": grouped("groups2"), "groups20": grouped("groups20"),
                        "torch_foreach": torch_step("foreach"), "torch_fused": torch_step("fused")}
            for fn in variants.values():
                for _ in range(args.warmup):
                    fn()
            torch.cuda.synchronize()
            times = {k: [] for k in variants}
            for _ in range(args.rounds):
                for k, fn in variants.items():
                    times[k].append(timed(fn, args.steps))
            out = {}
            for k, ts in times.items():
                ts = sorted(ts)
                us = ts[len(ts) // 2]
                bps = BYTES_PER_PARAM[optimizer] * sum(numels) / (us * 1e-6)
                out[k] = {"us_per_step_median": round(us, 1), "us_per_step_min": round(ts[0], 1), "us_per_step_max": round(ts[-1], 1)}
                if not k.startswith("torch"):
                    out[k]["achieved_tb_per_s"] = round(bps / 1e12, 3)
                    out[k]["share_of_datasheet_hbm_bw"] = round(bps / DATASHEET_HBM_BPS, 3)
            for k in ("groups2", "groups20"):
                out[f"{k}_over_fused_time"] = round(out[k]["us_per_step_median"] / out["fused"]["us_per_step_median"], 4)
            row[optimizer] = out
            del opts, tparams, state
        results["optimizer"][model] = row
        assert comm.status() == 0
        del views, flat_p, flat_g
        comm.close()
        torch.cuda.empty_cache()


def end_to_end(args, results):
    from bagua_net_b200.parallel import BnetDDP, no_weight_decay_groups

    x = torch.randn(args.batch, 3, 224, 224, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (args.batch,), device="cuda")
    engines = {}
    for name in ("sgd", "sgd_no_decay_groups"):
        torch.manual_seed(0)
        model = build_model("resnet50").cuda().to(torch.bfloat16).to(memory_format=torch.channels_last)
        groups = no_weight_decay_groups(model) if name != "sgd" else None
        eng = BnetDDP(model, lr=LR, momentum=MU, weight_decay=WD, bucket_mb=64.0, param_groups=groups)
        eng.enable_cuda_graph(True)
        for _ in range(args.warmup):
            eng.train_step(x, y)
        engines[name] = eng
    torch.cuda.synchronize()
    imgs = {k: [] for k in engines}
    for _ in range(args.e2e_rounds):
        for k, eng in engines.items():
            us = timed(lambda: eng.train_step(x, y), args.e2e_steps)
            imgs[k].append(args.batch / (us * 1e-6))
    for k, v in imgs.items():
        v = sorted(v)
        results["end_to_end"][k] = {"img_per_s_median": round(v[len(v) // 2], 1), "img_per_s_min": round(v[0], 1),
                                    "img_per_s_max": round(v[-1], 1)}
    results["end_to_end"]["groups_over_plain_img_per_s"] = round(
        results["end_to_end"]["sgd_no_decay_groups"]["img_per_s_median"] / results["end_to_end"]["sgd"]["img_per_s_median"], 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/param_groups_step")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--e2e-steps", type=int, default=30)
    ap.add_argument("--e2e-rounds", type=int, default=5)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("param_groups_step.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    results = {"card": card(), "bucket_mb": 64, "param_dtype": "bf16", "steps_per_window": args.steps, "rounds": args.rounds,
               "bytes_per_param": BYTES_PER_PARAM, "datasheet_hbm_tb_per_s": DATASHEET_HBM_BPS / 1e12, "optimizer": {},
               "end_to_end": {}}
    optimizer_times(args, results)
    if not args.no_e2e:
        end_to_end(args, results)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "param_groups_step.json"), "w") as f:
        json.dump(results, f, indent=1)
    print(json.dumps(results))


if __name__ == "__main__":
    main()

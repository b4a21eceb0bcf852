"""Data-parallel VGG16 training on the fused path: backward overlaps ONE kernel per gradient bucket that all-reduces,
applies SGD to this rank's fp32 shard and broadcasts the new bf16 parameters (bagua_net_b200.parallel.BnetDDP).
The workload is the reference's headline benchmark (reference README.md:52-84), with synthetic ImageNet-shaped data."""
import argparse
import os

import torch

from bagua_net_b200.models import build_model
from bagua_net_b200.parallel import BnetDDP, init_process_group_from_env, no_weight_decay_groups


def batches(n, batch, device_rank):
    g = torch.Generator().manual_seed(1234 + device_rank)
    for _ in range(n):
        yield (torch.randn(batch, 3, 224, 224, generator=g).bfloat16().pin_memory(),
               torch.randint(0, 1000, (batch,), generator=g).pin_memory())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--batch", type=int, default=32, help="images per rank and optimizer step")
    ap.add_argument("--accumulation-steps", type=int, default=1,
                    help="split every batch into this many micro-batches (one forward/backward each) and update once")
    ap.add_argument("--ema-decay", type=float, default=None,
                    help="keep an exponential moving average of the weights with this decay (torchvision uses 0.99998)")
    ap.add_argument("--ema-every", type=int, default=1, help="update the EMA after every this many optimizer steps")
    ap.add_argument("--no-decay-1d", action="store_true",
                    help="no weight decay on biases and normalisation weights (torchvision's --norm-weight-decay 0.0)")
    ap.add_argument("--model", default="vgg16")
    ap.add_argument("--checkpoint", default="", help="save the model and the whole optimizer state here at the end")
    ap.add_argument("--resume", default="",
                    help="start from a --checkpoint file, saved at any number of GPUs (every rank loads it)")
    a = ap.parse_args()
    init_process_group_from_env()
    rank = int(os.environ.get("RANK", "0"))
    model = build_model(a.model, fused=True).cuda().bfloat16().to(memory_format=torch.channels_last)
    engine = BnetDDP(model, lr=0.01, momentum=0.9, weight_decay=1e-4, accumulation_steps=a.accumulation_steps,
                     ema_decay=a.ema_decay, ema_every=a.ema_every,
                     param_groups=no_weight_decay_groups(model) if a.no_decay_1d else None)
    engine.enable_cuda_graph(True)            # forward + backward + every bucket kernel replay as one graph
    engine.set_lr(0.01)                       # hyper-parameters live in device memory: the graph follows the schedule
    first = 0
    if a.resume:
        ck = torch.load(a.resume, map_location="cpu")
        model.load_state_dict(ck["model"])
        engine.load_full_optimizer_state_dict(ck["optimizer"])   # this rank's shards, whatever the saving world size
        first = ck.get("step", 0)
        if rank == 0:
            print(f"resumed from {a.resume} at step {first}")
    last = []

    def remember(it):                         # (the last batch, for the evaluation on the EMA weights below)
        for b in it:
            last[:] = [b]
            yield b

    for step, loss in enumerate(engine.train_from_host(remember(batches(a.steps, a.batch, rank))), start=first):
        if step % 10 == 0:
            engine.set_lr(0.01 * 0.5 ** (step // 20))
            if rank == 0:
                print(f"step {step:4d}  loss {float(loss):.4f}")
    if a.ema_decay is not None and last:
        x, y = last[0][0].cuda().contiguous(memory_format=torch.channels_last), last[0][1].cuda()
        model.eval()
        with engine.ema_parameters(), torch.no_grad():    # every rank takes part
            ema_loss = float(torch.nn.functional.cross_entropy(model(x).float(), y))
        model.train()
        if rank == 0:
            print(f"last batch on the EMA weights: loss {ema_loss:.4f}")
    if a.checkpoint:
        state = engine.full_optimizer_state_dict()            # collective: rank 0 gets the whole state, the others None
        if rank == 0:
            torch.save({"model": model.state_dict(), "optimizer": state, "step": first + a.steps}, a.checkpoint)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""NVLink peer bandwidth of the transport executor (K1) and of the fused ops (K4/K5):
rank 0 pushes from its own heap into rank 1's heap through the same sm_90a cluster kernels
that serve the plugin's isend.  Launch with torchrun on >= 2 GPUs.

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 bench/p2p_bw.py
Env: BNET_COPY_ENGINE=ldst|tma  BNET_NCLUSTERS  BNET_CLUSTER_SIZE  BNET_PERSISTENT
"""
import os
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bagua_net_b200.ops import P2PExecutor  # noqa: E402
from bagua_net_b200.parallel import SymmComm, init_process_group_from_env  # noqa: E402


def main():
    init_process_group_from_env("nccl")
    rank, world = dist.get_rank(), dist.get_world_size()
    comm = SymmComm(1 << 30)
    ex = P2PExecutor(torch.cuda.current_device())
    maxb = 256 << 20
    src = comm.alloc(maxb, torch.uint8)
    dst = comm.alloc(maxb, torch.uint8)
    src.random_(0, 255)
    torch.cuda.synchronize()
    dist.barrier()
    peer = (rank + 1) % world
    remote = comm.peer_tensor(dst, peer)
    rows = []
    if rank == 0:
        for op, elt in (("copy", 1), ("red_add_f32", 4), ("acc_bf16_to_f32", 2)):
            for nbytes in (64 << 10, 512 << 10, 4 << 20, 32 << 20, 256 << 20):
                if op == "acc_bf16_to_f32" and nbytes * 2 > maxb:
                    continue
                s = src[:nbytes].view(torch.uint8)
                d = remote
                if op == "red_add_f32":
                    s, d = src[:nbytes].view(torch.float32), remote[:nbytes].view(torch.float32)
                elif op == "acc_bf16_to_f32":
                    s, d = src[:nbytes].view(torch.bfloat16), remote[:2 * nbytes].view(torch.float32)
                else:
                    d = remote[:nbytes]
                ex.run(op, s, d)
                iters = 20 if nbytes <= (32 << 20) else 5
                t0 = time.perf_counter()
                tickets = [ex.submit(op, s, d, sync=False) for _ in range(iters)]
                for t in tickets:
                    ex.wait(t)
                dt = (time.perf_counter() - t0) / iters
                rows.append((op, nbytes, dt * 1e6, nbytes / dt / 1e9))
                print(f"{op:18s} {nbytes:>10d} B  {dt * 1e6:9.1f} us  {nbytes / dt / 1e9:8.1f} GB/s (src bytes over NVLink to GPU {peer})", flush=True)
    dist.barrier()
    # correctness of the last plain copy as seen by the receiver
    if rank == 0:
        ex.run("copy", src[:1 << 20], remote[:1 << 20])
    torch.cuda.synchronize()
    dist.barrier()
    lst = [torch.zeros(1, device="cuda", dtype=torch.float64) for _ in range(world)]
    dist.all_gather(lst, src[:1 << 20].double().sum().reshape(1))
    if rank == 1:
        assert float(dst[:1 << 20].double().sum()) == float(lst[0]), "peer copy mismatch"
        print("peer copy verified on the receiving GPU", flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

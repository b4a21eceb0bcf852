"""Tensor-parallel linear layers whose collective is fused into the GEMM kernel (csrc/cuda/tc_gemm.cu; `BNET_TC=0` disables):

  row-parallel     y = sum_r x[:, K_r] @ w[:, K_r].T        epilogue adds every tile into all ranks' outputs (all-reduce)
  reduce-scatter   same, each rank keeps its row block       epilogue sends a tile only to its owner
  all-gather       y = [x_0; x_1; ...] @ w.T                 peers' row shards are TMA-loaded over NVLink as operands

The kernel checks itself against an fp32 reference on this GPU before it is used (`tc_linear.self_check`); the row-parallel
variant is covered by `tests/test_gpu.py::test_tcgen05_row_parallel_linear_2gpu`."""
import torch

from bagua_net_b200.ops import tc_linear
from bagua_net_b200.parallel import SymmComm, init_process_group_from_env


def main():
    init_process_group_from_env()
    comm = SymmComm(256 << 20)
    if not (tc_linear.enabled() and tc_linear.self_check(verbose=comm.rank == 0)):
        if comm.rank == 0:
            print("wgmma path disabled (BNET_TC=0), unsupported on this GPU, or its self-check failed")
        return
    M, N, K = 512, 4096, 8192
    torch.manual_seed(0)
    x_full = torch.randn(M, K, device="cuda").bfloat16()
    w_full = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
    kr = K // comm.world
    x_k, w_k = x_full[:, comm.rank * kr:(comm.rank + 1) * kr], w_full[:, comm.rank * kr:(comm.rank + 1) * kr]
    y = tc_linear.row_parallel_linear(x_k, w_k, comm)                   # fp32 [M, N] on every rank
    ys = tc_linear.linear_reduce_scatter(x_k, w_k, comm)                # fp32 [M / world, N]
    rows = M // comm.world
    shard = comm.alloc(rows * K, torch.bfloat16).view(rows, K)
    shard.copy_(x_full[comm.rank * rows:(comm.rank + 1) * rows])
    yg = tc_linear.allgather_linear(shard, w_full, comm)                # bf16 [M, N]
    ref = x_full.float() @ w_full.float().t()
    torch.cuda.synchronize()
    if comm.rank == 0:
        print("row-parallel max err", float((y - ref).abs().max()), " reduce-scatter", float((ys - ref[:rows]).abs().max()),
              " all-gather", float((yg.float() - ref).abs().max()), " watchdog", tc_linear.last_error())


if __name__ == "__main__":
    main()

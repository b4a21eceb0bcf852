/*
 * bnet tensor-core linear — wgmma / TMA GEMM with a fused epilogue, optionally fused with the all-reduce
 * of a row-parallel (tensor-parallel) linear layer.
 *
 *   out[M,N] = act(x[M,K] . w[N,K]^T + bias[N])                       bnet_tc_linear        (bf16 in, bf16 out)
 *   outs[r][M,N] += x[M,K] . w[N,K]^T (+ bias)   for every rank r      bnet_tc_linear_reduce (bf16 in, fp32 out)
 *
 * The second form is the "GEMM -> all-reduce in ONE kernel" of a row-parallel layer: every rank multiplies its K-shard
 * and the epilogue adds the fp32 tile straight into the symmetric-heap output of EVERY rank — one multimem.red per
 * vector through the NVSwitch multicast mapping, or one red.global per peer over NVLink — so the transfer of tile t
 * overlaps the math of tile t+1.  The caller zeroes the output, runs a rank barrier before and after (bnet_barrier).
 *
 * The reference has no counterpart (it moves bytes for NCCL; SURVEY.md §2.6): this is the GPU "compute step followed
 * by a collective" path (on by default, BNET_TC=0 disables); descriptor packing is checked against the CuTe definitions on
 * the host (tests/test_utils.py), and every launch carries a watchdog that turns a stuck pipeline into an error code
 * instead of a hang.  Callers in Python trust the kernels only after a self-check on the GPU at hand (ops/tc_linear.py,
 * ops/tc_conv.py).
 */
#ifndef BNET_TC_H_
#define BNET_TC_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { BNET_TC_ACT_NONE = 0, BNET_TC_ACT_RELU = 1 };
#define BNET_TC_MAX_OUTS 16
#define BNET_TC_MAX_PEERS 8

/* 1 when the driver exposes cuTensorMapEncodeTiled and the current device is compute capability 9.x (sm_90a) */
int bnet_tc_supported(void);

/* How a problem is tiled (pure host function; also used by the tests).  Returns 0 and fills the plan, or -1. */
typedef struct BnetTcPlan {
  int swap;       /* 1: w rows fill the 128 accumulator rows and x rows are the MMA N dimension (small batch) */
  int bn;         /* MMA N (tile width of the other operand): 32 / 64 (swapped), 128 or 256 */
  int stages;     /* TMA -> MMA shared-memory pipeline depth */
  int grid_x, grid_y, grid_z;   /* tiles along the column operand, tiles along the lane operand, K slices */
  int smem_bytes;
  int k_blocks;   /* 64-element K blocks in total */
  int k_per_split;
  int ctas;       /* CTAs launched per K slice: min(tiles, SMs / K slices); each walks tiles ctas apart (persistent) */
} BnetTcPlan;
int bnet_tc_plan(int M, int N, int K, int reduce, int splits, BnetTcPlan* plan);

/* err_dev: one int in device memory, 0 before the launch; non-zero afterwards = the watchdog tripped (value = role). */
int bnet_tc_linear(const void* x, const void* w, const void* bias, void* out, int M, int N, int K, int ldx, int ldw,
                   int ldo, int act, int* err_dev, void* stream);

/* Split-K for weight-streaming (small batch) layers with the finish fused into the kernel: K is cut into `splits` slices
 * so that every SM streams weights; partial tiles meet as fp32 adds in `ws` ([M, N] floats), and the slice that arrives
 * last at a tile (counted in `counters`, one int per output tile plus one) applies bias / activation and writes the bf16 result.
 * `ws` and `counters` must be all zero on entry and are all zero again on exit.  One launch. */
int bnet_tc_linear_splitk(const void* x, const void* w, const void* bias, void* out, float* ws, int* counters, int M, int N, int K,
                          int ldx, int ldw, int ldo, int act, int splits, int* err_dev, void* stream);

/* outs: n_outs device pointers to fp32 [M, ldo] buffers (this rank's mapping of every rank's output), or ONE multicast
 * pointer when multicast != 0.  splits > 1 additionally splits K over grid.z (the adds make it free). */
int bnet_tc_linear_reduce(const void* x, const void* w, const void* bias, void* const* outs, int n_outs, int multicast,
                          int M, int N, int K, int ldx, int ldw, int ldo, int splits, int* err_dev, void* stream);

/* all-gather -> GEMM: the activation is sharded by rows over n_shards ranks (rows_per_shard a multiple of 128);
 * x_shards[r] is this rank's mapping of rank r's shard (symmetric heap).  out[n_shards * rows_per_shard, N], bf16. */
int bnet_tc_allgather_linear(const void* const* x_shards, int n_shards, int rows_per_shard, const void* w, const void* bias,
                             void* out, int N, int K, int ldx, int ldw, int ldo, int act, int* err_dev, void* stream);

/* GEMM -> reduce-scatter: like bnet_tc_linear_reduce, but rank r's output (outs[r], fp32 [M / n_ranks, ldo]) receives
 * only the rows it owns.  M must divide by n_ranks. */
int bnet_tc_linear_reduce_scatter(const void* x, const void* w, const void* bias, void* const* outs, int n_ranks, int M, int N,
                                  int K, int ldx, int ldw, int ldo, int splits, int* err_dev, void* stream);

/* The two backward GEMMs of the same layer, without materialising any transpose (the operands whose reduction dimension
 * is the outer one are staged as MN-major tiles):
 *   dx[M,K] = gy[M,N] . w[N,K]            dw[N,K] = gy[M,N]^T . x[M,K]   (N > 64)
 * bf16 in, fp32 accumulate, bf16 out. */
int bnet_tc_linear_dgrad(const void* gy, const void* w, void* dx, int M, int N, int K, int ldgy, int ldw, int lddx, int* err_dev,
                         void* stream);
int bnet_tc_linear_wgrad(const void* gy, const void* x, void* dw, int M, int N, int K, int ldgy, int ldx, int lddw, int* err_dev,
                         void* stream);

/* 3x3 / stride 1 / pad 1 convolution as an implicit GEMM on the same kernel: the 128 accumulator rows of a tile are a
 * patch of output pixels whose (shifted) inputs arrive as 4-D TMA boxes of the NHWC activation — padding = the TMA unit's
 * zero fill — and bias + ReLU are applied in the epilogue.  bf16 NHWC activations, filters [Cout][3][3][Cin] (the memory of a
 * channels_last torch Conv2d weight).  Cin % 64 == 0, Cout % 8 == 0.  dgrad reads the SAME filter MN-major with flipped
 * taps (Cin % 64 == 0 and Cout % 64 == 0). */
int bnet_tc_conv3x3(const void* x, const void* w, const void* bias, void* out, int N, int H, int W, int Cin, int Cout, int act,
                    int* err_dev, void* stream);
int bnet_tc_conv3x3_dgrad(const void* gy, const void* w, void* dx, int N, int H, int W, int Cin, int Cout, int* err_dev,
                          void* stream);
/* Filter gradient dw[Cout][3][3][Cin] (bf16) of the same convolution: D[co, tap * Cin + ci] = sum over pixels of
 * gy[p, co] * x[p + tap, ci] — both operands MN-major 4-D TMA boxes of 64 pixels, the pixel blocks split over grid.z, the
 * slice that arrives last at a tile converts the fp32 sums (split-K fix-up).  `ws`: fp32 [Cout][9 Cin], `counters`:
 * bnet_tc_conv3x3_wgrad_tiles(Cin, Cout) ints; both all zero on entry and all zero again on exit.  splits <= 0: automatic.
 * Cin % 64 == 0, Cout % 64 == 0. */
int bnet_tc_conv3x3_wgrad(const void* gy, const void* x, void* dw, float* ws, int* counters, int N, int H, int W, int Cin, int Cout,
                          int splits, int* err_dev, void* stream);
int bnet_tc_conv3x3_wgrad_tiles(int Cin, int Cout);
int bnet_tc_conv3x3_wgrad_plan(int N, int H, int W, int Cin, int Cout, int splits, BnetTcPlan* plan);   /* host only */
/* The tiling of bnet_tc_conv3x3 (dgrad = 0: Cred = Cin, Cn = Cout) or bnet_tc_conv3x3_dgrad (dgrad = 1: Cred = Cout, Cn = Cin);
 * patch = {bw, bh, bn}: one 128-row tile is bw x bh pixels of bn images.  Host only. */
int bnet_tc_conv3x3_plan(int N, int H, int W, int Cred, int Cn, int dgrad, BnetTcPlan* plan, int patch[3]);

/* The 64-bit wgmma shared-memory matrix descriptor (K-major, 128-byte swizzle) the kernel issues, exposed so a host test
 * can compare it with the CuTe definition. */
uint64_t bnet_tc_smem_desc(uint32_t smem_addr);
uint64_t bnet_tc_smem_desc_mn(uint32_t smem_addr);            /* MN-major tile staged as 64 x 64 boxes */

const char* bnet_tc_last_error(void);

#ifdef __cplusplus
}
#endif
#endif

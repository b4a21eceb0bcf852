// Fused memory-bound layers of the benchmark models (channels_last / NHWC), sm_90a.
//
// In an eager VGG16 bf16 step, bias-add, ReLU, max-pool, their backward passes and the bias-gradient
// reductions are all HBM-bound, one full pass over the activations each.  These kernels fuse every such
// chain behind a convolution into ONE pass:
//   forward : z = conv(x,w)  ->  y = relu(z + b)                      (in place, 1 read + 1 write)
//             z = conv(x,w)  ->  p = maxpool2x2(relu(z + b)), idx      (y is never materialised)
//   backward: gz = gy * (y > 0)  and  gb = sum(gz)                     (1 pass instead of 2.3)
//             gz = scatter(gp, idx) and gb = sum(gp | valid)           (1 pass instead of 3+,
//                                                                      uint8 indices instead of int64)
// All accesses are 16-byte vectors along the contiguous channel dimension.  The per-thread walks live in
// nn_body.cuh so that `make test` can run them over an emulated grid on the CPU (csrc/tests/nn_emu_test.cc).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "core/common.h"
#include "cuda/nn_body.cuh"

#define BNET_API extern "C" __attribute__((visibility("default")))

namespace bnet {
namespace nn {

// ---- y = relu(z + b), in place ------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) bias_relu_kernel(T* __restrict__ z, const T* __restrict__ bias, size_t nvec, int cvec) {
  bias_relu_thread<T>(z, bias, nvec, cvec, (size_t)blockIdx.x * blockDim.x + threadIdx.x, (size_t)gridDim.x * blockDim.x);
}

// block-wide reduction of per-thread channel-group sums; the block stores its partial sums at row blockIdx.x (pitch `ld`
// floats) of `part`, and sum_rows_kernel adds the rows up in block order.  Atomics would add them in whatever order the
// blocks finish, and the gradient would then differ in its last bits from run to run.
template <int V>
__device__ __forceinline__ void reduce_bias_grad(float* acc, float* __restrict__ part, int ld, int cvec, float* smem) {
  const int rows = blockDim.x / cvec;           // threads that share a channel group
  const int grp = threadIdx.x % cvec, trow = threadIdx.x / cvec;
#pragma unroll
  for (int k = 0; k < V; k++) smem[(trow * cvec + grp) * V + k] = acc[k];
  __syncthreads();
  if (trow == 0) {
    float s[V];
#pragma unroll
    for (int k = 0; k < V; k++) s[k] = 0.f;
    for (int r = 0; r < rows; r++)
#pragma unroll
      for (int k = 0; k < V; k++) s[k] += smem[(r * cvec + grp) * V + k];
    float* row = part + (size_t)blockIdx.x * ld + grp * V;
#pragma unroll
    for (int k = 0; k < V; k += 4) *reinterpret_cast<float4*>(row + k) = make_float4(s[k], s[k + 1], s[k + 2], s[k + 3]);
  }
}

// dst[c] += sum of part[b * ld + c] over b < nrows, in a fixed order: a block takes 32 columns, its 8 warps the rows
// b = warp (mod 8) in ascending order, and warp 0 adds the 8 sums up in warp order
__global__ void __launch_bounds__(256) sum_rows_kernel(const float* __restrict__ part, float* __restrict__ dst, int nrows, int ld) {
  __shared__ float sums[8][32];
  const int cx = threadIdx.x & 31, g = threadIdx.x >> 5, c = blockIdx.x * 32 + cx;
  float v = 0.f;
  if (c < ld)
    for (int b = g; b < nrows; b += 8) v += part[(size_t)b * ld + c];
  sums[g][cx] = v;
  __syncthreads();
  if (g == 0 && c < ld) {
    float t = sums[0][cx];
#pragma unroll
    for (int k = 1; k < 8; k++) t += sums[k][cx];
    dst[c] += t;
  }
}

// ---- gz = gy * (y > 0) ; gb += column sums of gz ---------------------------------------------------
// blockDim.x is a multiple of cvec; the per-thread walk (4 rows = 8 x 16-byte loads in flight) is nn_body.cuh.
template <typename T>
__global__ void __launch_bounds__(256) relu_bwd_bias_grad_kernel(const T* __restrict__ gy, const T* __restrict__ y,
                                                                 T* __restrict__ gz, float* __restrict__ gb, size_t rows,
                                                                 int cvec) {
  constexpr int V = Vec<T>::N;
  extern __shared__ float smem[];
  float acc[V];
#pragma unroll
  for (int k = 0; k < V; k++) acc[k] = 0.f;
  relu_bwd_thread<T, 4>(gy, y, gz, rows, cvec, blockDim.x / cvec, threadIdx.x % cvec, threadIdx.x / cvec, blockIdx.x,
                        gridDim.x, acc);
  reduce_bias_grad<V>(acc, gb, cvec * V, cvec, smem);
}

// ---- p = maxpool2x2(relu(z + b)) with a 1-byte index per element ---------------------------------
template <typename T>
__global__ void __launch_bounds__(256) bias_relu_pool_fwd_kernel(const T* __restrict__ z, const T* __restrict__ bias,
                                                                 T* __restrict__ p, uint8_t* __restrict__ idx, int N, int H,
                                                                 int W, int cvec) {
  bias_relu_pool_fwd_thread<T>(z, bias, p, idx, N, H, W, cvec, (size_t)blockIdx.x * blockDim.x + threadIdx.x,
                               (size_t)gridDim.x * blockDim.x);
}

// ---- gz = scatter(gp through idx) ; gb += sum of routed gradients -----------------------------------
template <typename T>
__global__ void __launch_bounds__(256) pool_relu_bwd_bias_grad_kernel(const T* __restrict__ gp, const uint8_t* __restrict__ idx,
                                                                      T* __restrict__ gz, float* __restrict__ gb, int N, int H,
                                                                      int W, int cvec) {
  constexpr int V = Vec<T>::N;
  extern __shared__ float smem[];
  float acc[V];
#pragma unroll
  for (int k = 0; k < V; k++) acc[k] = 0.f;
  pool_relu_bwd_thread<T, 4>(gp, idx, gz, N, H, W, cvec, blockDim.x / cvec, threadIdx.x % cvec, threadIdx.x / cvec,
                             blockIdx.x, gridDim.x, acc);
  reduce_bias_grad<V>(acc, gb, cvec * V, cvec, smem);
}

// ---- BatchNorm (training) + ReLU + residual, four kernels (see nn_body.cuh) ------------------------------------
template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16(v); }

template <typename T>
__global__ void __launch_bounds__(256) bn_stats_kernel(const T* __restrict__ z, float* __restrict__ stats, size_t rows, int cvec) {
  constexpr int V = Vec<T>::N;
  extern __shared__ float smem[];
  float acc[2 * V];
#pragma unroll
  for (int k = 0; k < 2 * V; k++) acc[k] = 0.f;
  bn_stats_thread<T, 4>(z, rows, cvec, blockDim.x / cvec, threadIdx.x % cvec, threadIdx.x / cvec, blockIdx.x, gridDim.x, acc);
  const int C = cvec * V;
  reduce_bias_grad<V>(acc, stats, 2 * C, cvec, smem);          // sum
  __syncthreads();
  reduce_bias_grad<V>(acc + V, stats + C, 2 * C, cvec, smem);  // sum of squares
}

// y = relu?(bn(z) (+ res)); block 0 also updates the running statistics (unbiased variance, PyTorch semantics)
template <typename T>
__global__ void __launch_bounds__(256) bn_apply_kernel(const T* __restrict__ z, const T* __restrict__ res, T* __restrict__ y,
                                                       const float* __restrict__ stats, const T* __restrict__ gamma,
                                                       const T* __restrict__ beta, T* __restrict__ running_mean,
                                                       T* __restrict__ running_var, size_t rows, int cvec, float eps,
                                                       float momentum, int relu) {
  constexpr int V = Vec<T>::N;
  const int C = cvec * V, grp = threadIdx.x % cvec, trow = threadIdx.x / cvec;
  float mean[V], invstd[V], var[V], scale[V], shift[V];
  bn_moments<V>(stats, C, grp, 1.0f / (float)rows, eps, mean, invstd, var);
#pragma unroll
  for (int k = 0; k < V; k++) {
    const int c = grp * V + k;
    scale[k] = to_f<T>(gamma[c]) * invstd[k];
    shift[k] = to_f<T>(beta[c]) - mean[k] * scale[k];
  }
  if (blockIdx.x == 0 && trow == 0 && running_mean) {
    const float unbias = rows > 1 ? (float)rows / (float)(rows - 1) : 1.0f;
#pragma unroll
    for (int k = 0; k < V; k++) {
      const int c = grp * V + k;
      running_mean[c] = from_f<T>((1.f - momentum) * to_f<T>(running_mean[c]) + momentum * mean[k]);
      running_var[c] = from_f<T>((1.f - momentum) * to_f<T>(running_var[c]) + momentum * var[k] * unbias);
    }
  }
  bn_apply_thread<T, 4>(z, res, y, rows, cvec, blockDim.x / cvec, grp, trow, blockIdx.x, gridDim.x, scale, shift, relu != 0);
}

template <typename T>
__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(const T* __restrict__ gy, const T* __restrict__ y,
                                                            const T* __restrict__ z, const float* __restrict__ stats,
                                                            float* __restrict__ gsum, size_t rows, int cvec, float eps, int relu) {
  constexpr int V = Vec<T>::N;
  extern __shared__ float smem[];
  const int C = cvec * V, grp = threadIdx.x % cvec, trow = threadIdx.x / cvec;
  float mean[V], invstd[V], var[V], acc[2 * V];
  bn_moments<V>(stats, C, grp, 1.0f / (float)rows, eps, mean, invstd, var);
#pragma unroll
  for (int k = 0; k < 2 * V; k++) acc[k] = 0.f;
  bn_bwd_reduce_thread<T, 2>(gy, y, z, rows, cvec, blockDim.x / cvec, grp, trow, blockIdx.x, gridDim.x, mean, invstd, relu != 0, acc);
  reduce_bias_grad<V>(acc, gsum, 2 * C, cvec, smem);            // s1 = sum dy
  __syncthreads();
  reduce_bias_grad<V>(acc + V, gsum + C, 2 * C, cvec, smem);    // s2 = sum dy * xhat
}

// gz, gres, and (block 0) the parameter gradients dgamma = s2, dbeta = s1
template <typename T>
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const T* __restrict__ gy, const T* __restrict__ y,
                                                           const T* __restrict__ z, T* __restrict__ gz, T* __restrict__ gres,
                                                           const float* __restrict__ stats, const float* __restrict__ gsum,
                                                           const T* __restrict__ gamma, T* __restrict__ dgamma,
                                                           T* __restrict__ dbeta, size_t rows, int cvec, float eps, int relu) {
  constexpr int V = Vec<T>::N;
  const int C = cvec * V, grp = threadIdx.x % cvec, trow = threadIdx.x / cvec;
  const float inv_m = 1.0f / (float)rows;
  float mean[V], invstd[V], var[V], a[V], c1[V], c2[V];
  bn_moments<V>(stats, C, grp, inv_m, eps, mean, invstd, var);
#pragma unroll
  for (int k = 0; k < V; k++) {
    const int c = grp * V + k;
    a[k] = to_f<T>(gamma[c]) * invstd[k];
    c1[k] = gsum[c] * inv_m;
    c2[k] = gsum[C + c] * inv_m;
  }
  if (blockIdx.x == 0 && trow == 0) {
#pragma unroll
    for (int k = 0; k < V; k++) {
      const int c = grp * V + k;
      dbeta[c] = from_f<T>(gsum[c]);
      dgamma[c] = from_f<T>(gsum[C + c]);
    }
  }
  bn_bwd_apply_thread<T, 2>(gy, y, z, gz, gres, rows, cvec, blockDim.x / cvec, grp, trow, blockIdx.x, gridDim.x, mean, invstd, a,
                            c1, c2, relu != 0);
}

}  // namespace nn
}  // namespace bnet

using namespace bnet::nn;

// SMs of the current device; 132 (H100 SXM) when there is none to ask
static int sm_count() {
  static const int n = [] {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0)
      return v;
    (void)cudaGetLastError();
    return 132;
  }();
  return n;
}

static int nn_grid_cap() {
  static const int cap = [] {
    long long v = bnet::env_int("NN_BLOCKS_PER_SM", 2);
    if (v < 1) v = 1;
    if (v > 16) v = 16;
    return (int)v * sm_count();
  }();
  return cap;
}

// dst[0 .. ld) += the `rows` partial rows the reduce kernel left in `part`
static int finish_rows(const float* part, float* dst, int rows, int ld, cudaStream_t st) {
  if (cudaGetLastError() != cudaSuccess) return -2;
  sum_rows_kernel<<<(ld + 31) / 32, 256, 0, st>>>(part, dst, rows, ld);
  return cudaGetLastError() == cudaSuccess ? 1 : -2;
}

// Rows of the workspace `part` the reduce entry points below may use: the caller passes part with at least this many rows
// of C (bias gradients) or 2 C (BatchNorm sums) floats, e.g. a tensor allocated on the stream of the call.
BNET_API int bnet_nn_partial_rows(void) { return nn_grid_cap(); }

// dtype: 0 = f32, 1 = bf16 (same codes as bnet_coll.h).  All tensors NHWC-contiguous, C % vec == 0.
// Return 1 (the fused pass was launched) or <0.
BNET_API int bnet_nn_bias_relu(void* z, const void* bias, long long rows, int C, int dtype, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int V = dtype == 1 ? 8 : 4;
  if (C % V) return -1;
  size_t nvec = (size_t)rows * C / V;
  int grid = (int)((nvec + 255) / 256 < sm_count() * 16 ? (nvec + 255) / 256 : sm_count() * 16);
  if (grid < 1) grid = 1;
  if (dtype == 1) bias_relu_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((__nv_bfloat16*)z, (const __nv_bfloat16*)bias, nvec, C / V);
  else bias_relu_kernel<float><<<grid, 256, 0, st>>>((float*)z, (const float*)bias, nvec, C / V);
  return cudaGetLastError() == cudaSuccess ? 1 : -2;
}

BNET_API int bnet_nn_relu_bwd_bias_grad(const void* gy, const void* y, void* gz, float* gb, float* part, long long rows, int C, int dtype,
                                        void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int V = dtype == 1 ? 8 : 4;
  if (C % V || C / V > 256) return -1;
  const int cvec = C / V;
  const int threads = (256 / cvec) * cvec;
  const int rpb = threads / cvec;
  // at least 8 rows per thread before another block is worth its partial row (small late layers: few rows, many channels)
  long long want = (rows + 8LL * rpb - 1) / (8LL * rpb);
  int grid = (int)(want < nn_grid_cap() ? want : nn_grid_cap());
  if (grid < 1) grid = 1;
  if (!part) return -1;
  size_t smem = (size_t)threads * V * sizeof(float);
  if (dtype == 1)
    relu_bwd_bias_grad_kernel<__nv_bfloat16><<<grid, threads, smem, st>>>((const __nv_bfloat16*)gy, (const __nv_bfloat16*)y,
                                                                       (__nv_bfloat16*)gz, part, (size_t)rows, cvec);
  else
    relu_bwd_bias_grad_kernel<float><<<grid, threads, smem, st>>>((const float*)gy, (const float*)y, (float*)gz, part, (size_t)rows, cvec);
  return finish_rows(part, gb, grid, C, st);
}

BNET_API int bnet_nn_bias_relu_pool_fwd(const void* z, const void* bias, void* p, void* idx, int N, int H, int W, int C, int dtype,
                                        void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int V = dtype == 1 ? 8 : 4;
  if (C % V || (H & 1) || (W & 1)) return -1;
  size_t total = (size_t)N * (H / 2) * (W / 2) * (C / V);
  int grid = (int)((total + 255) / 256 < sm_count() * 16 ? (total + 255) / 256 : sm_count() * 16);
  if (grid < 1) grid = 1;
  if (dtype == 1)
    bias_relu_pool_fwd_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>((const __nv_bfloat16*)z, (const __nv_bfloat16*)bias,
                                                                  (__nv_bfloat16*)p, (uint8_t*)idx, N, H, W, C / V);
  else
    bias_relu_pool_fwd_kernel<float><<<grid, 256, 0, st>>>((const float*)z, (const float*)bias, (float*)p, (uint8_t*)idx, N, H, W, C / V);
  return cudaGetLastError() == cudaSuccess ? 1 : -2;
}

BNET_API int bnet_nn_pool_relu_bwd_bias_grad(const void* gp, const void* idx, void* gz, float* gb, float* part, int N, int H, int W, int C,
                                             int dtype, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int V = dtype == 1 ? 8 : 4;
  if (C % V || C / V > 256 || (H & 1) || (W & 1)) return -1;
  const int cvec = C / V;
  const int threads = (256 / cvec) * cvec;
  const int rpb = threads / cvec;
  long long rows = (long long)N * (H / 2) * (W / 2);
  // at least 8 rows per thread before another block is worth its partial row (small late layers: few rows, many channels)
  long long want = (rows + 8LL * rpb - 1) / (8LL * rpb);
  int grid = (int)(want < nn_grid_cap() ? want : nn_grid_cap());
  if (grid < 1) grid = 1;
  if (!part) return -1;
  size_t smem = (size_t)threads * V * sizeof(float);
  if (dtype == 1)
    pool_relu_bwd_bias_grad_kernel<__nv_bfloat16><<<grid, threads, smem, st>>>((const __nv_bfloat16*)gp, (const uint8_t*)idx,
                                                                            (__nv_bfloat16*)gz, part, N, H, W, cvec);
  else
    pool_relu_bwd_bias_grad_kernel<float><<<grid, threads, smem, st>>>((const float*)gp, (const uint8_t*)idx, (float*)gz, part, N, H, W, cvec);
  return finish_rows(part, gb, grid, C, st);
}


// ---- BatchNorm family.  stats / gsum: 2*C floats ([sum | sumsq], [s1 | s2]) that the caller zeroes before the
// reduce kernels.  gamma/beta/running stats have the activation dtype.  res, running_*, gres may be NULL.
namespace {
struct RowGrid { int threads, grid; size_t smem; };
RowGrid row_grid(long long rows, int cvec, int V, int accs) {
  RowGrid g;
  g.threads = (256 / cvec) * cvec;
  const int rpb = g.threads / cvec;
  // at least 8 rows per thread before another block is worth its partial row (small late layers: few rows, many channels)
  long long want = (rows + 8LL * rpb - 1) / (8LL * rpb);
  // the element-wise kernels (accs == 0) leave no partial rows: they keep the larger grid
  const int cap = accs ? nn_grid_cap() : sm_count() * 8;
  g.grid = (int)(want < cap ? want : cap);
  if (g.grid < 1) g.grid = 1;
  g.smem = (size_t)g.threads * V * sizeof(float) * (accs ? 1 : 0);
  return g;
}
}  // namespace

BNET_API int bnet_nn_bn_stats(const void* z, float* stats, float* part, long long rows, int C, int dtype, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int V = dtype == 1 ? 8 : 4;
  if (C % V || C / V > 256 || rows < 1) return -1;
  const RowGrid g = row_grid(rows, C / V, V, 1);
  if (!part) return -1;
  if (dtype == 1) bn_stats_kernel<__nv_bfloat16><<<g.grid, g.threads, g.smem, st>>>((const __nv_bfloat16*)z, part, (size_t)rows, C / V);
  else bn_stats_kernel<float><<<g.grid, g.threads, g.smem, st>>>((const float*)z, part, (size_t)rows, C / V);
  return finish_rows(part, stats, g.grid, 2 * C, st);
}

BNET_API int bnet_nn_bn_apply(const void* z, const void* res, void* y, const float* stats, const void* gamma, const void* beta,
                              void* running_mean, void* running_var, long long rows, int C, float eps, float momentum, int relu,
                              int dtype, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int V = dtype == 1 ? 8 : 4;
  if (C % V || C / V > 256 || rows < 1) return -1;
  const RowGrid g = row_grid(rows, C / V, V, 0);
  if (dtype == 1)
    bn_apply_kernel<__nv_bfloat16><<<g.grid, g.threads, 0, st>>>((const __nv_bfloat16*)z, (const __nv_bfloat16*)res, (__nv_bfloat16*)y, stats,
                                                                (const __nv_bfloat16*)gamma, (const __nv_bfloat16*)beta,
                                                                (__nv_bfloat16*)running_mean, (__nv_bfloat16*)running_var, (size_t)rows,
                                                                C / V, eps, momentum, relu);
  else
    bn_apply_kernel<float><<<g.grid, g.threads, 0, st>>>((const float*)z, (const float*)res, (float*)y, stats, (const float*)gamma,
                                                        (const float*)beta, (float*)running_mean, (float*)running_var, (size_t)rows, C / V,
                                                        eps, momentum, relu);
  return cudaGetLastError() == cudaSuccess ? 1 : -2;
}

BNET_API int bnet_nn_bn_bwd_reduce(const void* gy, const void* y, const void* z, const float* stats, float* gsum, float* part, long long rows,
                                   int C, float eps, int relu, int dtype, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int V = dtype == 1 ? 8 : 4;
  if (C % V || C / V > 256 || rows < 1) return -1;
  const RowGrid g = row_grid(rows, C / V, V, 1);
  if (!part) return -1;
  if (dtype == 1)
    bn_bwd_reduce_kernel<__nv_bfloat16><<<g.grid, g.threads, g.smem, st>>>((const __nv_bfloat16*)gy, (const __nv_bfloat16*)y,
                                                                          (const __nv_bfloat16*)z, stats, part, (size_t)rows, C / V, eps, relu);
  else
    bn_bwd_reduce_kernel<float><<<g.grid, g.threads, g.smem, st>>>((const float*)gy, (const float*)y, (const float*)z, stats, part,
                                                                  (size_t)rows, C / V, eps, relu);
  return finish_rows(part, gsum, g.grid, 2 * C, st);
}

BNET_API int bnet_nn_bn_bwd_apply(const void* gy, const void* y, const void* z, void* gz, void* gres, const float* stats,
                                  const float* gsum, const void* gamma, void* dgamma, void* dbeta, long long rows, int C, float eps,
                                  int relu, int dtype, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int V = dtype == 1 ? 8 : 4;
  if (C % V || C / V > 256 || rows < 1) return -1;
  const RowGrid g = row_grid(rows, C / V, V, 0);
  if (dtype == 1)
    bn_bwd_apply_kernel<__nv_bfloat16><<<g.grid, g.threads, 0, st>>>((const __nv_bfloat16*)gy, (const __nv_bfloat16*)y, (const __nv_bfloat16*)z,
                                                                    (__nv_bfloat16*)gz, (__nv_bfloat16*)gres, stats, gsum,
                                                                    (const __nv_bfloat16*)gamma, (__nv_bfloat16*)dgamma, (__nv_bfloat16*)dbeta,
                                                                    (size_t)rows, C / V, eps, relu);
  else
    bn_bwd_apply_kernel<float><<<g.grid, g.threads, 0, st>>>((const float*)gy, (const float*)y, (const float*)z, (float*)gz, (float*)gres,
                                                            stats, gsum, (const float*)gamma, (float*)dgamma, (float*)dbeta, (size_t)rows,
                                                            C / V, eps, relu);
  return cudaGetLastError() == cudaSuccess ? 1 : -2;
}

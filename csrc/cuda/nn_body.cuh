// Per-thread bodies of the fused NHWC layer kernels (csrc/cuda/nn_kernels.cu).
//
// Every kernel is "one thread walks a strided set of 16-byte channel vectors"; the walk is written here as a
// plain function of (block, thread) so that the SAME code is (a) inlined into the __global__ kernels by nvcc
// and (b) compiled by g++ and driven over an emulated grid by csrc/tests/nn_emu_test.cc — the CPU check of
// the indexing, masking and index-coding logic that `make test` runs without a GPU.
//
// Memory-level parallelism rule used below: issue ALL the 16-byte
// loads of an unrolled batch as raw vectors first, convert/compute afterwards.  Converting right after each
// load makes the next load wait behind the first one's latency and leaves the kernel at ~30% of HBM bandwidth.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define BNET_HD __host__ __device__ __forceinline__
#else
#define BNET_HD inline
#endif

namespace bnet {
namespace nn {

// ---- 16-byte streaming accesses (read-once / write-once data: do not allocate in L1) -------------------
BNET_HD int4 ld_stream(const int4* p) {
#if defined(__CUDA_ARCH__)
  int4 r;
  asm("ld.global.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
#else
  return *p;
#endif
}
BNET_HD float4 ld_stream(const float4* p) {
#if defined(__CUDA_ARCH__)
  float4 r;
  asm("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
#else
  return *p;
#endif
}
BNET_HD void st_stream(int4* p, const int4& v) {
#if defined(__CUDA_ARCH__)
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
#else
  *p = v;
#endif
}
BNET_HD void st_stream(float4* p, const float4& v) {
#if defined(__CUDA_ARCH__)
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
#else
  *p = v;
#endif
}

// ---- one 16-byte vector of T as V floats ------------------------------------------------------------------
template <typename T> struct Vec;
template <> struct Vec<__nv_bfloat16> {
  static constexpr int N = 8;
  using Raw = int4;
  using Code = uint2;     // 8 one-byte pool codes
  static BNET_HD void unpack(const Raw& v, float* f) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int i = 0; i < 4; i++) { float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  }
  static BNET_HD Raw pack(const float* f) {
    Raw v;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
    for (int i = 0; i < 4; i++) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    return v;
  }
};
template <> struct Vec<float> {
  static constexpr int N = 4;
  using Raw = float4;
  using Code = uint32_t;  // 4 one-byte pool codes
  static BNET_HD void unpack(const Raw& v, float* f) { f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w; }
  static BNET_HD Raw pack(const float* f) { return make_float4(f[0], f[1], f[2], f[3]); }
};

template <typename T> BNET_HD typename Vec<T>::Raw load_raw(const T* p) {
  return *reinterpret_cast<const typename Vec<T>::Raw*>(p);
}
template <typename T> BNET_HD typename Vec<T>::Raw load_raw_stream(const T* p) {
  return ld_stream(reinterpret_cast<const typename Vec<T>::Raw*>(p));
}
template <typename T> BNET_HD void store_raw(T* p, const typename Vec<T>::Raw& v) {
  *reinterpret_cast<typename Vec<T>::Raw*>(p) = v;
}
template <typename T> BNET_HD void store_raw_stream(T* p, const typename Vec<T>::Raw& v) {
  st_stream(reinterpret_cast<typename Vec<T>::Raw*>(p), v);
}

// ---- ReLU as eager torch computes it: relu(NaN) = NaN (fmaxf would return 0 and hide a diverged run), and the backward
// passes the gradient unless y <= 0 (threshold_backward), so a NaN activation passes it too
BNET_HD float relu(float v) { return v <= 0.f ? 0.f : v; }
BNET_HD bool relu_passes(float y) { return !(y <= 0.f); }

// ---- y = relu(z + b), in place ---------------------------------------------------------------------------------
// gtid/gthreads: global thread index / number of threads in the grid.  nvec = rows * cvec 16-byte vectors.
template <typename T>
BNET_HD void bias_relu_thread(T* z, const T* bias, size_t nvec, int cvec, size_t gtid, size_t gthreads) {
  constexpr int V = Vec<T>::N;
  for (size_t i = gtid; i < nvec; i += gthreads) {
    float v[V], b[V];
    Vec<T>::unpack(load_raw(z + i * V), v);
    Vec<T>::unpack(load_raw(bias + (i % cvec) * V), b);
#pragma unroll
    for (int k = 0; k < V; k++) v[k] = relu(v[k] + b[k]);
    store_raw(z + i * V, Vec<T>::pack(v));
  }
}

// ---- p = maxpool2x2(relu(z + b)) with a 1-byte code per element ------------------------------------------------
// code: bits 0-1 = position of the max inside the window (dy*2+dx), bit 2 = the gradient flows (relu_passes(max)).
// The window follows torch's max_pool2d: the first maximum wins a tie, and a NaN wins over any number (a later NaN over an
// earlier one), so the pooled value is NaN and the gradient goes to that element.
template <typename T>
BNET_HD void bias_relu_pool_fwd_thread(const T* z, const T* bias, T* p, uint8_t* idx, int N, int H, int W, int cvec,
                                       size_t gtid, size_t gthreads) {
  constexpr int V = Vec<T>::N;
  const int Ho = H / 2, Wo = W / 2;
  const size_t total = (size_t)N * Ho * Wo * cvec;
  for (size_t i = gtid; i < total; i += gthreads) {
    const int g = (int)(i % cvec);
    size_t t = i / cvec;
    const int wo = (int)(t % Wo);
    t /= Wo;
    const int ho = (int)(t % Ho);
    const int n = (int)(t / Ho);
    const size_t base = (((size_t)n * H + 2 * ho) * W + 2 * wo) * cvec + g;   // in vectors
    typename Vec<T>::Raw raw[4];
    raw[0] = load_raw(z + base * V);
    raw[1] = load_raw(z + (base + cvec) * V);
    raw[2] = load_raw(z + (base + (size_t)W * cvec) * V);
    raw[3] = load_raw(z + (base + (size_t)W * cvec + cvec) * V);
    float v[4][V], b[V];
#pragma unroll
    for (int q = 0; q < 4; q++) Vec<T>::unpack(raw[q], v[q]);
    Vec<T>::unpack(load_raw(bias + (size_t)g * V), b);
    float out[V];
    typename Vec<T>::Code codes;
    uint8_t* code = reinterpret_cast<uint8_t*>(&codes);
#pragma unroll
    for (int k = 0; k < V; k++) {
      float m = v[0][k] + b[k];
      int a = 0;
#pragma unroll
      for (int q = 1; q < 4; q++) {
        const float u = v[q][k] + b[k];
        if (u > m || u != u) { m = u; a = q; }
      }
      out[k] = relu(m);
      code[k] = (uint8_t)(a | (relu_passes(m) ? 4 : 0));
    }
    store_raw(p + i * V, Vec<T>::pack(out));
    *reinterpret_cast<typename Vec<T>::Code*>(idx + i * V) = codes;
  }
}

// ---- gz = relu_passes(y) ? gy : 0 ; acc += this thread's column sums of gz -------------------------------------------------
// rows = N*H*W, cvec = C / V.  The block owns rpb = threads/cvec consecutive rows per step; thread (trow, grp)
// always sees channel group grp.  U rows per thread are loaded (2*U 16-byte requests in flight) before any
// dependent work; out-of-range rows of the last batch re-read row r0 (valid) instead of branching.
template <typename T, int U>
BNET_HD void relu_bwd_thread(const T* gy, const T* y, T* gz, size_t rows, int cvec, int rpb, int grp, int trow,
                             size_t block, size_t nblocks, float* acc) {
  constexpr int V = Vec<T>::N;
  using Raw = typename Vec<T>::Raw;
  const size_t step = nblocks * (size_t)rpb;
  for (size_t r0 = block * rpb + trow; r0 < rows; r0 += U * step) {
    Raw g[U], a[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t r = r0 + u * step;
      const size_t off = ((r < rows ? r : r0) * cvec + grp) * V;
      g[u] = load_raw_stream(gy + off);
      a[u] = load_raw_stream(y + off);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t r = r0 + u * step;
      if (r < rows) {
        float gf[V], af[V];
        Vec<T>::unpack(g[u], gf);
        Vec<T>::unpack(a[u], af);
#pragma unroll
        for (int k = 0; k < V; k++) {
          gf[k] = relu_passes(af[k]) ? gf[k] : 0.f;
          acc[k] += gf[k];
        }
        store_raw_stream(gz + (r * cvec + grp) * V, Vec<T>::pack(gf));
      }
    }
  }
}

// ---- gz = scatter(gp through the pool codes) ; acc += this thread's sums of the routed gradients ------------
// rows = N*(H/2)*(W/2) pooled positions; same thread/row mapping as relu_bwd_thread.
template <typename T, int U>
BNET_HD void pool_relu_bwd_thread(const T* gp, const uint8_t* idx, T* gz, int N, int H, int W, int cvec, int rpb,
                                  int grp, int trow, size_t block, size_t nblocks, float* acc) {
  constexpr int V = Vec<T>::N;
  using Raw = typename Vec<T>::Raw;
  using Code = typename Vec<T>::Code;
  const int Ho = H / 2, Wo = W / 2;
  const size_t rows = (size_t)N * Ho * Wo;
  const size_t step = nblocks * (size_t)rpb;
  for (size_t r0 = block * rpb + trow; r0 < rows; r0 += U * step) {
    Raw graw[U];
    Code craw[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t r = r0 + u * step;
      const size_t i = (r < rows ? r : r0) * cvec + grp;
      graw[u] = load_raw_stream(gp + i * V);
      craw[u] = *reinterpret_cast<const Code*>(idx + i * V);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t r = r0 + u * step;
      if (r >= rows) continue;
      size_t t = r;
      const int wo = (int)(t % Wo);
      t /= Wo;
      const int ho = (int)(t % Ho);
      const int n = (int)(t / Ho);
      float gv[V];
      Vec<T>::unpack(graw[u], gv);
      const uint8_t* code = reinterpret_cast<const uint8_t*>(&craw[u]);
      float o[4][V];
#pragma unroll
      for (int k = 0; k < V; k++) {
        const float gk = (code[k] & 4) ? gv[k] : 0.f;
        acc[k] += gk;
#pragma unroll
        for (int q = 0; q < 4; q++) o[q][k] = ((code[k] & 3) == q) ? gk : 0.f;
      }
      const size_t base = (((size_t)n * H + 2 * ho) * W + 2 * wo) * cvec + grp;
      store_raw_stream(gz + base * V, Vec<T>::pack(o[0]));
      store_raw_stream(gz + (base + cvec) * V, Vec<T>::pack(o[1]));
      store_raw_stream(gz + (base + (size_t)W * cvec) * V, Vec<T>::pack(o[2]));
      store_raw_stream(gz + (base + (size_t)W * cvec + cvec) * V, Vec<T>::pack(o[3]));
    }
  }
}

// ==== training-mode BatchNorm fused with what follows it in a ResNet block ===========================================
//   forward : z = conv(x, w)                         (library call)
//             stats  = per-channel sum, sum of squares of z - K, K = z[row 0]               (bn_stats, 1 read)
//             y      = relu?( (z - mean) * invstd * gamma + beta  (+ residual) )            (bn_apply, 1-2 reads, 1 write)
//   backward: dy     = relu? (relu_passes(y) ? gy : 0) : gy
//             s1, s2 = per-channel sum of dy, of dy * xhat        (xhat = (z - mean) * invstd)  (bn_bwd_reduce)
//             gz     = gamma * invstd * (dy - s1/M - xhat * s2/M) ;  gres = dy              (bn_bwd_apply)
// Same thread/row mapping as relu_bwd_thread: thread (trow, grp) always sees channel group grp, so its channel
// constants live in registers for the whole walk.

// The statistics are sums of d = z - K with a per-channel pivot K, the channel's value in row 0.  Plain sums of z and z^2
// would give var = E[z^2] - mean^2, whose fp32 rounding error grows as (mean / std)^2 * 2^-24 (0.4 relative at
// mean / std = 1024); d is of the order of std, so var = E[d^2] - E[d]^2 keeps its error near 2^-24 at any offset.
// A NaN or infinite pivot makes every d, and so the channel's statistics, NaN (as eager torch's are).
template <typename T> BNET_HD void bn_pivot(const T* z, int grp, float* pivot) {
  Vec<T>::unpack(load_raw(z + (size_t)grp * Vec<T>::N), pivot);
}

// mean / inverse standard deviation of this thread's V channels from the shifted sums (biased variance); a NaN variance
// stays NaN (the clamp only lifts a rounding-negative value to 0)
template <int V>
BNET_HD void bn_moments(const float* stats, const float* pivot, int C, int grp, float inv_m, float eps, float* mean, float* invstd,
                        float* var) {
#pragma unroll
  for (int k = 0; k < V; k++) {
    const int c = grp * V + k;
    const float d = stats[c] * inv_m;
    float v = stats[C + c] * inv_m - d * d;
    v = v < 0.f ? 0.f : v;
    mean[k] = pivot[k] + d;
    var[k] = v;
#if defined(__CUDA_ARCH__)
    invstd[k] = rsqrtf(v + eps);
#else
    invstd[k] = 1.0f / sqrtf(v + eps);
#endif
  }
}

// acc[0..V) += z - pivot ; acc[V..2V) += (z - pivot)^2
template <typename T, int U>
BNET_HD void bn_stats_thread(const T* z, size_t rows, int cvec, int rpb, int grp, int trow, size_t block, size_t nblocks,
                             const float* pivot, float* acc) {
  constexpr int V = Vec<T>::N;
  using Raw = typename Vec<T>::Raw;
  const size_t step = nblocks * (size_t)rpb;
  for (size_t r0 = block * rpb + trow; r0 < rows; r0 += U * step) {
    Raw raw[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t r = r0 + u * step;
      raw[u] = load_raw_stream(z + ((r < rows ? r : r0) * cvec + grp) * V);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (r0 + u * step < rows) {
        float f[V];
        Vec<T>::unpack(raw[u], f);
#pragma unroll
        for (int k = 0; k < V; k++) {
          const float d = f[k] - pivot[k];
          acc[k] += d;
          acc[V + k] += d * d;
        }
      }
    }
  }
}

// y = relu?( (z - mean) * scale + beta (+ res) ) with per-channel mean, scale = gamma * invstd and beta held by the thread.
// (z * scale + (beta - mean * scale) would save a subtraction but round z * scale, an error of 2^-24 |mean| * scale: far more
//  than the result's own rounding once |mean| is large next to std, and y = beta would not hold on a constant channel.)
template <typename T, int U>
BNET_HD void bn_apply_thread(const T* z, const T* res, T* y, size_t rows, int cvec, int rpb, int grp, int trow, size_t block,
                             size_t nblocks, const float* mean, const float* scale, const float* beta, bool relu) {
  constexpr int V = Vec<T>::N;
  using Raw = typename Vec<T>::Raw;
  const size_t step = nblocks * (size_t)rpb;
  for (size_t r0 = block * rpb + trow; r0 < rows; r0 += U * step) {
    Raw zr[U], rr[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t r = r0 + u * step;
      const size_t off = ((r < rows ? r : r0) * cvec + grp) * V;
      zr[u] = load_raw_stream(z + off);
      if (res) rr[u] = load_raw_stream(res + off);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t r = r0 + u * step;
      if (r < rows) {
        float f[V], q[V];
        Vec<T>::unpack(zr[u], f);
        if (res) Vec<T>::unpack(rr[u], q);
#pragma unroll
        for (int k = 0; k < V; k++) {
          float v = (f[k] - mean[k]) * scale[k] + beta[k];
          if (res) v += q[k];
          f[k] = relu ? bnet::nn::relu(v) : v;
        }
        store_raw_stream(y + (r * cvec + grp) * V, Vec<T>::pack(f));
      }
    }
  }
}

// acc[0..V) += dy ; acc[V..2V) += dy * xhat
template <typename T, int U>
BNET_HD void bn_bwd_reduce_thread(const T* gy, const T* y, const T* z, size_t rows, int cvec, int rpb, int grp, int trow,
                                  size_t block, size_t nblocks, const float* mean, const float* invstd, bool relu, float* acc) {
  constexpr int V = Vec<T>::N;
  using Raw = typename Vec<T>::Raw;
  const size_t step = nblocks * (size_t)rpb;
  for (size_t r0 = block * rpb + trow; r0 < rows; r0 += U * step) {
    Raw gr[U], yr[U], zr[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t r = r0 + u * step;
      const size_t off = ((r < rows ? r : r0) * cvec + grp) * V;
      gr[u] = load_raw_stream(gy + off);
      zr[u] = load_raw_stream(z + off);
      if (relu) yr[u] = load_raw_stream(y + off);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (r0 + u * step < rows) {
        float g[V], a[V], f[V];
        Vec<T>::unpack(gr[u], g);
        Vec<T>::unpack(zr[u], f);
        if (relu) Vec<T>::unpack(yr[u], a);
#pragma unroll
        for (int k = 0; k < V; k++) {
          const float dy = (!relu || relu_passes(a[k])) ? g[k] : 0.f;
          acc[k] += dy;
          acc[V + k] += dy * ((f[k] - mean[k]) * invstd[k]);
        }
      }
    }
  }
}

// gz = a * (dy - c1 - xhat * c2) with a = gamma * invstd, c1 = s1 / M, c2 = s2 / M ; gres = dy (when there is a residual)
template <typename T, int U>
BNET_HD void bn_bwd_apply_thread(const T* gy, const T* y, const T* z, T* gz, T* gres, size_t rows, int cvec, int rpb, int grp,
                                 int trow, size_t block, size_t nblocks, const float* mean, const float* invstd, const float* a,
                                 const float* c1, const float* c2, bool relu) {
  constexpr int V = Vec<T>::N;
  using Raw = typename Vec<T>::Raw;
  const size_t step = nblocks * (size_t)rpb;
  for (size_t r0 = block * rpb + trow; r0 < rows; r0 += U * step) {
    Raw gr[U], yr[U], zr[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t r = r0 + u * step;
      const size_t off = ((r < rows ? r : r0) * cvec + grp) * V;
      gr[u] = load_raw_stream(gy + off);
      zr[u] = load_raw_stream(z + off);
      if (relu) yr[u] = load_raw_stream(y + off);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t r = r0 + u * step;
      if (r < rows) {
        float g[V], act[V], f[V], o[V];
        Vec<T>::unpack(gr[u], g);
        Vec<T>::unpack(zr[u], f);
        if (relu) Vec<T>::unpack(yr[u], act);
#pragma unroll
        for (int k = 0; k < V; k++) {
          const float dy = (!relu || relu_passes(act[k])) ? g[k] : 0.f;
          g[k] = dy;
          o[k] = a[k] * (dy - c1[k] - (f[k] - mean[k]) * invstd[k] * c2[k]);
        }
        const size_t off = (r * cvec + grp) * V;
        store_raw_stream(gz + off, Vec<T>::pack(o));
        if (gres) store_raw_stream(gres + off, Vec<T>::pack(g));
      }
    }
  }
}

}  // namespace nn
}  // namespace bnet

// bnet collectives: symmetric-heap communicator + fused sm_90a kernels (K4/K5/K6).
//
//   * NVLS all-reduce: multimem.ld_reduce (reduction inside the NVSwitch) followed by
//     multimem.st (switch broadcast) on a cuMulticast mapping of the symmetric heap —
//     one kernel, no separate elementwise reduce launch, no host hop.
//   * P2P all-reduce: peer loads (reduce-scatter) + peer stores (all-gather) over NVLink.
//   * fused all-reduce + SGD + parameter broadcast: the gradient never makes a round trip
//     through HBM between "communication" and "optimizer"; optimizer state is sharded.
// Cross-rank synchronisation is a per-CTA flag handshake in the symmetric signal pad
// (release/acquire CAS at system scope) so CTAs of different ranks pair up directly.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <errno.h>
#include <poll.h>
#include <stdio.h>
#include <string.h>
#include <sys/socket.h>
#include <sys/un.h>
#include <unistd.h>

#include <string>
#include <thread>
#include <vector>

#include "bnet/bnet_coll.h"
#include "core/common.h"
#include "cuda/driver_api.h"
#include "cuda/ptx.cuh"

#define BNET_API extern "C" __attribute__((visibility("default")))

namespace bnet {
namespace coll {

constexpr int kThreads = 512;
constexpr size_t kPadBytes = 1 << 18;   // signal pad at the start of every rank's allocation
static_assert(BNET_COLL_SIGNAL_BYTES <= kPadBytes, "signal pad too small");

struct CollDev {
  char* heap[BNET_COLL_MAX_WORLD];   // every rank's allocation mapped here (own included)
  char* mc;                          // multicast alias of the allocations (nullptr without NVLS)
  uint32_t* status;                  // mapped host word: != 0 after a watchdog trip
  int rank, world;
};

thread_local std::string g_err;
static int fail(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
static int fail(const char* fmt, ...) {
  char b[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(b, sizeof(b), fmt, ap);
  va_end(ap);
  g_err = b;
  BNET_WARN("coll: %s", b);
  return -1;
}

// ------------------------------------------------------------------ device helpers
__device__ __forceinline__ uint32_t cas_release_sys(uint32_t* p, uint32_t cmp, uint32_t val) {
  uint32_t old;
  asm volatile("atom.global.release.sys.cas.b32 %0, [%1], %2, %3;" : "=r"(old) : "l"(p), "r"(cmp), "r"(val) : "memory");
  return old;
}
__device__ __forceinline__ uint32_t cas_acquire_sys(uint32_t* p, uint32_t cmp, uint32_t val) {
  uint32_t old;
  asm volatile("atom.global.acquire.sys.cas.b32 %0, [%1], %2, %3;" : "=r"(old) : "l"(p), "r"(cmp), "r"(val) : "memory");
  return old;
}

constexpr uint64_t kWatchdogNs = 20ull * 1000000000ull;

// CTA b of every rank meets CTA b of every other rank.  Writes issued before the barrier by any
// thread of the CTA are visible to the peers after it (bar.sync + release/acquire at sys scope).
__device__ __forceinline__ void rank_barrier(const CollDev& d, int chan) {
  __syncthreads();
  if ((int)threadIdx.x < d.world) {
    const int peer = threadIdx.x;
    const size_t idx = ((size_t)chan * BNET_COLL_MAX_BLOCKS + blockIdx.x) * BNET_COLL_MAX_WORLD;
    uint32_t* put = reinterpret_cast<uint32_t*>(d.heap[peer]) + idx + d.rank;
    uint32_t* get = reinterpret_cast<uint32_t*>(d.heap[d.rank]) + idx + peer;
    const uint64_t t0 = ptx::globaltimer();
    while (cas_release_sys(put, 0u, 1u) != 0u) {
      if (ptx::globaltimer() - t0 > kWatchdogNs) { *d.status = 1; break; }
    }
    while (cas_acquire_sys(get, 1u, 0u) != 1u) {
      if (ptx::globaltimer() - t0 > kWatchdogNs) { *d.status = 2; break; }
    }
  }
  __syncthreads();
}

template <int DT> struct VecTraits;
template <> struct VecTraits<BNET_F32> { static constexpr int kElems = 4; };
template <> struct VecTraits<BNET_BF16> { static constexpr int kElems = 8; };
template <> struct VecTraits<BNET_F16> { static constexpr int kElems = 8; };

// 16-byte vector <-> fp32 lanes
template <int DT>
__device__ __forceinline__ void unpack(const int4& v, float* f) {
  if constexpr (DT == BNET_F32) {
    f[0] = __int_as_float(v.x); f[1] = __int_as_float(v.y); f[2] = __int_as_float(v.z); f[3] = __int_as_float(v.w);
  } else if constexpr (DT == BNET_BF16) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int i = 0; i < 4; i++) { float2 t = __bfloat1622float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  } else {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; i++) { float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  }
}
template <int DT>
__device__ __forceinline__ int4 pack(const float* f) {
  int4 v;
  if constexpr (DT == BNET_F32) {
    v.x = __float_as_int(f[0]); v.y = __float_as_int(f[1]); v.z = __float_as_int(f[2]); v.w = __float_as_int(f[3]);
  } else if constexpr (DT == BNET_BF16) {
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
    for (int i = 0; i < 4; i++) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  } else {
    __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; i++) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  }
  return v;
}

template <int OP>
__device__ __forceinline__ float combine(float a, float b) {
  if constexpr (OP == BNET_MAX) return fmaxf(a, b);
  else if constexpr (OP == BNET_MIN) return fminf(a, b);
  else return a + b;
}

// in-switch reduction of one 16-byte vector across all ranks bound to the multicast object
template <int DT, int OP>
__device__ __forceinline__ int4 mc_ld_reduce(const char* p) {
  int4 r;
  if constexpr (DT == BNET_F32) {
    static_assert(OP == BNET_SUM || OP == BNET_AVG, "multimem f32 supports add only");
    float4 f = ptx::multimem_ld_reduce_add_f32x4(p);
    r.x = __float_as_int(f.x); r.y = __float_as_int(f.y); r.z = __float_as_int(f.z); r.w = __float_as_int(f.w);
  } else if constexpr (DT == BNET_BF16) {
    if constexpr (OP == BNET_MAX)
      asm volatile("multimem.ld_reduce.relaxed.sys.global.max.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                   : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    else if constexpr (OP == BNET_MIN)
      asm volatile("multimem.ld_reduce.relaxed.sys.global.min.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                   : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    else
      r = ptx::multimem_ld_reduce_add_bf16x8(p);
  } else {
    if constexpr (OP == BNET_MAX)
      asm volatile("multimem.ld_reduce.relaxed.sys.global.max.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                   : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    else if constexpr (OP == BNET_MIN)
      asm volatile("multimem.ld_reduce.relaxed.sys.global.min.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                   : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    else
      r = ptx::multimem_ld_reduce_add_f16x8(p);
  }
  return r;
}

template <int DT>
__device__ __forceinline__ int4 scale_vec(const int4& v, float s) {
  float f[8];
  unpack<DT>(v, f);
#pragma unroll
  for (int i = 0; i < VecTraits<DT>::kElems; i++) f[i] *= s;
  return pack<DT>(f);
}

// reduce one vector over all peers with NVLink loads, fp32 accumulation, fixed order from `first`
template <int DT, int OP, int W>
__device__ __forceinline__ void p2p_reduce_w(const CollDev& d, size_t byte_off, int first, float* acc) {
  int4 v[W];
#pragma unroll
  for (int j = 0; j < W; j++) {
    int p = first + j;
    if (p >= W) p -= W;
    v[j] = ptx::ld_na_v4(reinterpret_cast<const int4*>(d.heap[p] + byte_off));   // all loads in flight first
  }
  unpack<DT>(v[0], acc);
#pragma unroll
  for (int j = 1; j < W; j++) {
    float f[8];
    unpack<DT>(v[j], f);
#pragma unroll
    for (int i = 0; i < VecTraits<DT>::kElems; i++) acc[i] = combine<OP>(acc[i], f[i]);
  }
}
template <int DT, int OP>
__device__ __forceinline__ void p2p_reduce(const CollDev& d, size_t byte_off, int first, float* acc) {
  switch (d.world) {   // warp-uniform; the common NVSwitch sizes are fully unrolled
    case 2: return p2p_reduce_w<DT, OP, 2>(d, byte_off, first, acc);
    case 4: return p2p_reduce_w<DT, OP, 4>(d, byte_off, first, acc);
    case 8: return p2p_reduce_w<DT, OP, 8>(d, byte_off, first, acc);
    default: break;
  }
  int p = first;
  unpack<DT>(ptx::ld_na_v4(reinterpret_cast<const int4*>(d.heap[p] + byte_off)), acc);
  for (int j = 1; j < d.world; j++) {
    if (++p >= d.world) p -= d.world;
    float f[8];
    unpack<DT>(ptx::ld_na_v4(reinterpret_cast<const int4*>(d.heap[p] + byte_off)), f);
#pragma unroll
    for (int i = 0; i < VecTraits<DT>::kElems; i++) acc[i] = combine<OP>(acc[i], f[i]);
  }
}

// ------------------------------------------------------------------ all-reduce kernels
template <int DT, int OP>
__global__ void __launch_bounds__(kThreads) bnet_allreduce_nvls_kernel(CollDev d, size_t off, size_t nvec, int chan) {
  rank_barrier(d, chan);
  const size_t per = nvec / d.world;
  char* base = d.mc + off + (size_t)d.rank * per * 16;
  const size_t stride = (size_t)gridDim.x * kThreads;
  const float s = 1.0f / (float)d.world;
  constexpr int U = 8;   // 8 in-switch reductions in flight per thread
  size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
  for (; i + (U - 1) * stride < per; i += U * stride) {
    int4 v[U];
#pragma unroll
    for (int u = 0; u < U; u++) v[u] = mc_ld_reduce<DT, OP>(base + (i + u * stride) * 16);
#pragma unroll
    for (int u = 0; u < U; u++) {
      if constexpr (OP == BNET_AVG) v[u] = scale_vec<DT>(v[u], s);
      ptx::multimem_st_v4(base + (i + u * stride) * 16, v[u]);
    }
  }
  for (; i < per; i += stride) {
    int4 v = mc_ld_reduce<DT, OP>(base + i * 16);
    if constexpr (OP == BNET_AVG) v = scale_vec<DT>(v, s);
    ptx::multimem_st_v4(base + i * 16, v);
  }
  rank_barrier(d, chan);
}

// Direct two-shot all-reduce: rank r reduces slice r with peer LOADS (reduce-scatter) and writes the
// result to every rank with peer STORES (all-gather).  Per GPU S(n-1)/n bytes in and out, full duplex.
// U vectors x W peers of loads are issued before the first dependent add (NVLink latency ~2-3 us).
template <int DT, int OP, int W, int U>
__device__ __forceinline__ void p2p_allreduce_body(const CollDev& d, size_t off, size_t per, size_t start) {
  constexpr int E = VecTraits<DT>::kElems;
  const size_t stride = (size_t)gridDim.x * kThreads;
  const float s = 1.0f / (float)W;
  size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
  for (; i < per; i += U * stride) {
    int4 v[U][W];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t ii = i + u * stride;
      if (ii < per) {
        const size_t bo = off + (start + ii) * 16;
#pragma unroll
        for (int j = 0; j < W; j++) {
          int p = d.rank + j;
          if (p >= W) p -= W;
          v[u][j] = ptx::ld_na_v4(reinterpret_cast<const int4*>(d.heap[p] + bo));
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t ii = i + u * stride;
      if (ii >= per) continue;
      const size_t bo = off + (start + ii) * 16;
      float acc[8], f[8];
      unpack<DT>(v[u][0], acc);
#pragma unroll
      for (int j = 1; j < W; j++) {
        unpack<DT>(v[u][j], f);
#pragma unroll
        for (int k = 0; k < E; k++) acc[k] = combine<OP>(acc[k], f[k]);
      }
      if constexpr (OP == BNET_AVG) {
#pragma unroll
        for (int k = 0; k < E; k++) acc[k] *= s;
      }
      const int4 out = pack<DT>(acc);
#pragma unroll
      for (int j = 0; j < W; j++) {
        int p = d.rank + j;
        if (p >= W) p -= W;
        ptx::st_na_v4(reinterpret_cast<int4*>(d.heap[p] + bo), out);
      }
    }
  }
}

template <int DT, int OP>
__global__ void __launch_bounds__(kThreads) bnet_allreduce_p2p_kernel(CollDev d, size_t off, size_t nvec, int chan) {
  rank_barrier(d, chan);
  const size_t per = nvec / d.world;
  const size_t start = (size_t)d.rank * per;
  if (d.world == 2) p2p_allreduce_body<DT, OP, 2, 4>(d, off, per, start);
  else if (d.world == 4) p2p_allreduce_body<DT, OP, 4, 4>(d, off, per, start);
  else if (d.world == 8) p2p_allreduce_body<DT, OP, 8, 2>(d, off, per, start);
  else {
    const size_t stride = (size_t)gridDim.x * kThreads;
    const float s = 1.0f / (float)d.world;
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < per; i += stride) {
      const size_t bo = off + (start + i) * 16;
      float acc[8];
      p2p_reduce<DT, OP>(d, bo, d.rank, acc);
      if constexpr (OP == BNET_AVG) {
#pragma unroll
        for (int k = 0; k < VecTraits<DT>::kElems; k++) acc[k] *= s;
      }
      const int4 out = pack<DT>(acc);
      for (int j = 0; j < d.world; j++) {
        int p = d.rank + j;
        if (p >= d.world) p -= d.world;
        ptx::st_na_v4(reinterpret_cast<int4*>(d.heap[p] + bo), out);
      }
    }
  }
  rank_barrier(d, chan);
}

template <int DT, int OP>
__global__ void __launch_bounds__(kThreads) bnet_allreduce_oneshot_kernel(CollDev d, size_t off, char* out, size_t nvec,
                                                                         int chan) {
  rank_barrier(d, chan);
  const size_t stride = (size_t)gridDim.x * kThreads;
  const float s = 1.0f / (float)d.world;
  for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < nvec; i += stride) {
    float acc[8];
    p2p_reduce<DT, OP>(d, off + i * 16, 0, acc);   // same order on every rank: bitwise identical results
    if constexpr (OP == BNET_AVG) {
#pragma unroll
      for (int k = 0; k < VecTraits<DT>::kElems; k++) acc[k] *= s;
    }
    *reinterpret_cast<int4*>(out + i * 16) = pack<DT>(acc);
  }
  rank_barrier(d, chan);   // inputs may be overwritten once every peer has read them
}

__global__ void __launch_bounds__(kThreads) bnet_barrier_kernel(CollDev d, int chan) { rank_barrier(d, chan); }


// ------------------------------------------------------------------ latency-optimal small all-reduce ("LL": flag in the data)
// No barrier at all: every 8-byte word a rank pushes to a peer carries 4 bytes of payload AND the call's epoch, so the
// arrival of the data IS its own signal (one NVLink store = one packet; an aligned 8-byte store is never torn).
//   ll area (same heap offset on every rank): [64-byte header][2 buffers][world senders][ll_words] x u64
//   header (read and written by the local rank only): {calls completed, blocks finished in the running call} — the call's
//   epoch is "completed + 1", read from DEVICE memory, so a captured CUDA graph replays correctly (every rank runs the
//   same sequence of calls on the area, so the epochs agree without ever being communicated)
//   push:  peer_ll[p][epoch & 1][my rank][i] = (epoch << 32) | my payload word i     for every peer p (own copy included)
//   pull:  spin on my_ll[epoch & 1][q][i] until its upper half == epoch, q = 0..world-1 in that fixed order (every rank
//          sums in the same order: bitwise identical results), accumulate in fp32, write out[i]
// Two buffers suffice: a rank cannot start call e+2 before every rank has pushed for e+1, i.e. finished reading call e.
// in / out are ordinary local pointers (any device memory, in place allowed): nothing but the ll area has to be symmetric.
template <int DT, int OP>
__device__ __forceinline__ void bnet_ll_word(const CollDev& d, size_t ll_off, size_t ll_words, const uint32_t* __restrict__ in,
                                             uint32_t* __restrict__ out, size_t i, size_t nelem, uint32_t epoch) {
  constexpr int EPW = (DT == BNET_F32) ? 1 : 2;          // elements per 4-byte word
  // my payload word (the last word of an odd-length 16-bit vector carries one element; the other half is zero)
  uint32_t w;
  if (EPW == 2 && (i + 1) * 2 > nelem) w = (uint32_t)reinterpret_cast<const uint16_t*>(in)[2 * i];
  else w = in[i];
  const uint64_t word = ((uint64_t)epoch << 32) | w;
  const size_t slot = ((size_t)(epoch & 1u) * d.world + d.rank) * ll_words + i;
  for (int j = 0; j < d.world; j++) {
    int p = d.rank + j;                                    // start with the own copy, then round the ring: spreads the links
    if (p >= d.world) p -= d.world;
    uint64_t* dst = reinterpret_cast<uint64_t*>(d.heap[p] + ll_off) + slot;
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" :: "l"(dst), "l"(word) : "memory");
  }
  float acc[2] = {0.f, 0.f};
  const uint64_t t0 = ptx::globaltimer();
  for (int q = 0; q < d.world; q++) {
    const uint64_t* src = reinterpret_cast<const uint64_t*>(d.heap[d.rank] + ll_off) + ((size_t)(epoch & 1u) * d.world + q) * ll_words + i;
    uint64_t v;
    for (;;) {
      asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(src) : "memory");
      if ((uint32_t)(v >> 32) == epoch) break;
      if (ptx::globaltimer() - t0 > kWatchdogNs) { *d.status = 3; break; }
    }
    const uint32_t pw = (uint32_t)v;
    float f[2];
    if constexpr (DT == BNET_F32) { f[0] = __uint_as_float(pw); f[1] = 0.f; }
    else if constexpr (DT == BNET_BF16) { f[0] = __uint_as_float(pw << 16); f[1] = __uint_as_float(pw & 0xffff0000u); }
    else { __half2 h = *reinterpret_cast<const __half2*>(&pw); float2 t = __half22float2(h); f[0] = t.x; f[1] = t.y; }
    if (q == 0) { acc[0] = f[0]; acc[1] = f[1]; }
    else { acc[0] = combine<OP>(acc[0], f[0]); acc[1] = combine<OP>(acc[1], f[1]); }
  }
  if constexpr (OP == BNET_AVG) { acc[0] *= 1.0f / (float)d.world; acc[1] *= 1.0f / (float)d.world; }
  if constexpr (DT == BNET_F32) {
    out[i] = __float_as_uint(acc[0]);
  } else {
    uint32_t r;
    if constexpr (DT == BNET_BF16) { __nv_bfloat162 h = __floats2bfloat162_rn(acc[0], acc[1]); r = *reinterpret_cast<uint32_t*>(&h); }
    else { __half2 h = __floats2half2_rn(acc[0], acc[1]); r = *reinterpret_cast<uint32_t*>(&h); }
    if ((i + 1) * 2 > nelem) reinterpret_cast<uint16_t*>(out)[2 * i] = (uint16_t)r;
    else out[i] = r;
  }
}

template <int DT, int OP>
__global__ void __launch_bounds__(256) bnet_allreduce_ll_kernel(CollDev d, size_t ll_hdr, size_t ll_words, const uint32_t* __restrict__ in,
                                                               uint32_t* __restrict__ out, size_t nwords, size_t nelem) {
  uint32_t* hdr = reinterpret_cast<uint32_t*>(d.heap[d.rank] + ll_hdr);
  const size_t ll_off = ll_hdr + 64;
  const uint32_t epoch = *(volatile uint32_t*)hdr + 1u;      // the same value in every block: hdr[0] moves only when ALL blocks are done
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nwords) bnet_ll_word<DT, OP>(d, ll_off, ll_words, in, out, i, nelem, epoch);
  // the last block to finish closes the call
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(hdr + 1, 1u) == gridDim.x - 1) {
      hdr[1] = 0;
      __threadfence();
      *(volatile uint32_t*)hdr = epoch;
    }
  }
}

// ------------------------------------------------------------------ fused all-reduce + SGD + broadcast
// MODE 0: single GPU, 1: NVLS multicast, 2: peer loads/stores
//
// One batch = U 16-byte gradient vectors per thread.  All loads of the batch (in-switch
// reductions / peer loads, fp32 master + momentum) are issued before any dependent math so that
// U*(1 + 2*E/4) requests per thread are in flight: the kernel is latency*bandwidth bound
// (NVLink round trip ~3 us, HBM), not ALU bound.
template <int DT, int MODE, int U>
__device__ __forceinline__ void fused_sgd_batch(const CollDev& d, size_t goff, size_t poff, size_t start, size_t i,
                                                size_t stride, float lr, float mu, float wd, float gscale,
                                                float* __restrict__ master, float* __restrict__ mom) {
  constexpr int E = VecTraits<DT>::kElems;
  constexpr int Q = E / 4;
  int4 gv[U];
  float4 pm[U][Q], bm[U][Q];
  float gp2p[(MODE == 2) ? U : 1][8];
#pragma unroll
  for (int u = 0; u < U; u++) {
    const size_t vo = (start + i + u * stride) * 16;
    if constexpr (MODE == 1) gv[u] = mc_ld_reduce<DT, BNET_SUM>(d.mc + goff + vo);
    else if constexpr (MODE == 2) p2p_reduce<DT, BNET_SUM>(d, goff + vo, d.rank, gp2p[u]);
    else gv[u] = ptx::ld_na_v4(reinterpret_cast<const int4*>(d.heap[0] + goff + vo));
  }
#pragma unroll
  for (int u = 0; u < U; u++) {
    const float4* mp = reinterpret_cast<const float4*>(master + (i + u * stride) * E);
    const float4* bp = reinterpret_cast<const float4*>(mom + (i + u * stride) * E);
#pragma unroll
    for (int q = 0; q < Q; q++) {
      pm[u][q] = ptx::ld_na_f4(mp + q);
      bm[u][q] = ptx::ld_na_f4(bp + q);
    }
  }
#pragma unroll
  for (int u = 0; u < U; u++) {
    const size_t vo = (start + i + u * stride) * 16;
    float g[8], p[8], b[8];
    if constexpr (MODE == 2) {
#pragma unroll
      for (int k = 0; k < E; k++) g[k] = gp2p[u][k];
    } else {
      unpack<DT>(gv[u], g);
    }
#pragma unroll
    for (int q = 0; q < Q; q++) {
      p[4 * q] = pm[u][q].x; p[4 * q + 1] = pm[u][q].y; p[4 * q + 2] = pm[u][q].z; p[4 * q + 3] = pm[u][q].w;
      b[4 * q] = bm[u][q].x; b[4 * q + 1] = bm[u][q].y; b[4 * q + 2] = bm[u][q].z; b[4 * q + 3] = bm[u][q].w;
    }
#pragma unroll
    for (int k = 0; k < E; k++) {
      float dp = fmaf(wd, p[k], g[k] * gscale);   // d_p = g/world + wd*p
      b[k] = fmaf(mu, b[k], dp);                  // buf = mu*buf + d_p
      p[k] = fmaf(-lr, b[k], p[k]);               // p  -= lr*buf
    }
    float4* mp = reinterpret_cast<float4*>(master + (i + u * stride) * E);
    float4* bp = reinterpret_cast<float4*>(mom + (i + u * stride) * E);
#pragma unroll
    for (int q = 0; q < Q; q++) {
      ptx::st_na_f4(mp + q, make_float4(p[4 * q], p[4 * q + 1], p[4 * q + 2], p[4 * q + 3]));
      ptx::st_na_f4(bp + q, make_float4(b[4 * q], b[4 * q + 1], b[4 * q + 2], b[4 * q + 3]));
    }
    const int4 out = pack<DT>(p);
    if constexpr (MODE == 1) {
      ptx::multimem_st_v4(d.mc + poff + vo, out);          // new parameters land on every rank
    } else if constexpr (MODE == 2) {
      for (int j = 0; j < d.world; j++) {
        int pr = d.rank + j;
        if (pr >= d.world) pr -= d.world;
        ptx::st_na_v4(reinterpret_cast<int4*>(d.heap[pr] + poff + vo), out);
      }
    } else {
      ptx::st_na_v4(reinterpret_cast<int4*>(d.heap[0] + poff + vo), out);
    }
  }
}

template <int DT, int MODE>
__global__ void __launch_bounds__(kThreads, 2) bnet_fused_sgd_kernel(CollDev d, size_t goff, size_t poff, size_t nvec,
                                                                 float lr, float mu, float wd, float gscale,
                                                                 float* __restrict__ master, float* __restrict__ mom,
                                                                 int zero_grads, int chan, const float* __restrict__ hp) {
  // hp != NULL: hyper-parameters {lr, momentum, weight decay, gradient scale} live in device memory, so a captured
  // CUDA graph keeps following a learning-rate schedule without being re-captured
  if (hp != nullptr) {
    lr = hp[0];
    mu = hp[1];
    wd = hp[2];
    gscale = hp[3];
  }
  if constexpr (MODE != 0) rank_barrier(d, chan);
  const size_t per = nvec / d.world;
  const size_t start = (size_t)d.rank * per;
  const size_t stride = (size_t)gridDim.x * kThreads;
  constexpr int U = 2;   // 16-byte gradient vectors per thread per batch (register budget: 2 CTAs/SM)
  size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
  for (; i + (U - 1) * stride < per; i += U * stride)
    fused_sgd_batch<DT, MODE, U>(d, goff, poff, start, i, stride, lr, mu, wd, gscale, master, mom);
  for (; i < per; i += stride)
    fused_sgd_batch<DT, MODE, 1>(d, goff, poff, start, i, stride, lr, mu, wd, gscale, master, mom);
  if constexpr (MODE != 0) rank_barrier(d, chan);
  if (zero_grads) {
    // Reset our gradients for the next backward.  The barrier above only pairs CTA b with CTA b of the peers (CTAs
    // of a grid start staggered when the kernel runs under backward on the side stream), so CTA b may only zero
    // what CTA b of some rank has READ: shard p, vectors p*per + i for exactly the i this CTA walks above.  Zeroing
    // with a flat index would hand vectors of shard p >= 1 to a different CTA than the one rank p reads them with.
    int4* gz = reinterpret_cast<int4*>(d.heap[d.rank] + goff);
    const int4 z = make_int4(0, 0, 0, 0);
    for (int p = 0; p < d.world; p++)
      for (size_t j = (size_t)blockIdx.x * kThreads + threadIdx.x; j < per; j += stride) ptx::st_na_v4(gz + (size_t)p * per + j, z);
    // vectors beyond per*world are read by nobody
    for (size_t j = per * d.world + (size_t)blockIdx.x * kThreads + threadIdx.x; j < nvec; j += stride) ptx::st_na_v4(gz + j, z);
  }
}

// ------------------------------------------------------------------ multi-tensor pack + cast (K5)
template <typename S, typename D>
__global__ void __launch_bounds__(256) bnet_pack_cast_kernel(const BnetPackItem* __restrict__ items, D* __restrict__ dst,
                                                            float scale) {
  const BnetPackItem it = items[blockIdx.y];
  const S* src = reinterpret_cast<const S*>(it.src);
  D* out = dst + it.dst_elem_off;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < it.numel; i += stride)
    out[i] = static_cast<D>(static_cast<float>(src[i]) * scale);
}

}  // namespace coll
}  // namespace bnet

// =====================================================================================
// host side
// =====================================================================================
using namespace bnet;
using namespace bnet::coll;
using bnet::cuda::driver;
using bnet::cuda::cu_err;

struct BnetColl {
  int rank = 0, world = 1, dev = 0;
  size_t alloc_bytes = 0;        // pad + heap, rounded to granularity
  size_t heap_bytes = 0;
  CUmemGenericAllocationHandle mem = 0;
  int mem_fd = -1;
  CUdeviceptr local_va = 0;
  CUdeviceptr peer_va[BNET_COLL_MAX_WORLD] = {0};
  CUmemGenericAllocationHandle peer_mem[BNET_COLL_MAX_WORLD] = {0};
  bool vmm = false;              // false: cudaMalloc fallback (single GPU without driver API)
  // multicast
  bool mc_supported = false, mc_ready = false;
  CUmemGenericAllocationHandle mc = 0;
  int mc_fd = -1;
  CUdeviceptr mc_va = 0;
  // fd server
  int srv_fd = -1;
  std::string uds_name;
  std::thread srv;
  uint32_t* status_host = nullptr;
  uint32_t* status_dev = nullptr;
  CollDev devp{};
};

namespace {

struct Blob {
  uint32_t magic;
  int32_t rank, dev;
  uint32_t pid;
  uint64_t alloc_bytes;
  uint32_t has_mc;
  uint32_t pad;
  char uds[64];
};
static_assert(sizeof(Blob) <= BNET_COLL_BLOB_BYTES, "blob");

int send_fd_msg(int sock, uint32_t tag, int fd) {
  msghdr mh{};
  iovec iov{&tag, sizeof(tag)};
  mh.msg_iov = &iov;
  mh.msg_iovlen = 1;
  char cbuf[CMSG_SPACE(sizeof(int))];
  memset(cbuf, 0, sizeof(cbuf));
  mh.msg_control = cbuf;
  mh.msg_controllen = sizeof(cbuf);
  cmsghdr* c = CMSG_FIRSTHDR(&mh);
  c->cmsg_level = SOL_SOCKET;
  c->cmsg_type = SCM_RIGHTS;
  c->cmsg_len = CMSG_LEN(sizeof(int));
  memcpy(CMSG_DATA(c), &fd, sizeof(int));
  ssize_t n;
  do { n = sendmsg(sock, &mh, MSG_NOSIGNAL); } while (n < 0 && errno == EINTR);
  return n == (ssize_t)sizeof(tag) ? 0 : -1;
}

int recv_fd_msg(int sock, uint32_t* tag, int* fd) {
  msghdr mh{};
  iovec iov{tag, sizeof(*tag)};
  mh.msg_iov = &iov;
  mh.msg_iovlen = 1;
  char cbuf[CMSG_SPACE(sizeof(int))];
  mh.msg_control = cbuf;
  mh.msg_controllen = sizeof(cbuf);
  *fd = -1;
  ssize_t n;
  do { n = recvmsg(sock, &mh, MSG_CMSG_CLOEXEC); } while (n < 0 && errno == EINTR);
  if (n != (ssize_t)sizeof(*tag)) return -1;
  for (cmsghdr* c = CMSG_FIRSTHDR(&mh); c; c = CMSG_NXTHDR(&mh, c))
    if (c->cmsg_level == SOL_SOCKET && c->cmsg_type == SCM_RIGHTS) memcpy(fd, CMSG_DATA(c), sizeof(int));
  return *fd >= 0 ? 0 : -1;
}

int map_handle(CUmemGenericAllocationHandle h, size_t bytes, int dev, CUdeviceptr* va_out) {
  const auto& d = driver();
  CUdeviceptr va = 0;
  CUresult r = d.MemAddressReserve(&va, bytes, 0, 0, 0);
  if (r != CUDA_SUCCESS) return fail("cuMemAddressReserve(%zu): %s", bytes, cu_err(r));
  if ((r = d.MemMap(va, bytes, 0, h, 0)) != CUDA_SUCCESS) {
    d.MemAddressFree(va, bytes);
    return fail("cuMemMap: %s", cu_err(r));
  }
  CUmemAccessDesc acc{};
  acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  acc.location.id = dev;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  if ((r = d.MemSetAccess(va, bytes, &acc, 1)) != CUDA_SUCCESS) {
    d.MemUnmap(va, bytes);
    d.MemAddressFree(va, bytes);
    return fail("cuMemSetAccess: %s", cu_err(r));
  }
  *va_out = va;
  return 0;
}

template <typename K, typename... Args>
int launch(K kernel, int nblocks, int threads, cudaStream_t st, Args... args) {
  kernel<<<nblocks, threads, 0, st>>>(args...);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("kernel launch failed: %s", cudaGetErrorString(e));
  return 1;
}

// Default CTA counts (BNET_COLL_BLOCKS_* override them): the in-switch (multimem) kernels only issue requests
// to the switch and get 32 CTAs; the peer load/store kernels get one CTA per SM of an H100 (132); a single GPU has
// no fabric to wait for but all of HBM to feed: 2 CTAs per SM.
enum BlockClass { BLK_NVLS = 0, BLK_P2P = 1, BLK_FUSED_NVLS = 2, BLK_SINGLE = 3 };
int pick_blocks(const BnetColl* c, size_t vec_per_rank, int requested, BlockClass cls) {
  if (requested > 0) return requested > BNET_COLL_MAX_BLOCKS ? BNET_COLL_MAX_BLOCKS : requested;
  static const int caps[4] = {(int)env_int("COLL_BLOCKS_NVLS", 32), (int)env_int("COLL_BLOCKS_P2P", 132),
                              (int)env_int("COLL_BLOCKS_FUSED_NVLS", 64), (int)env_int("COLL_BLOCKS_SINGLE", 264)};
  int cap = c->world == 1 ? caps[BLK_SINGLE] : caps[cls];
  if (cap > BNET_COLL_MAX_BLOCKS) cap = BNET_COLL_MAX_BLOCKS;
  if (cap < 1) cap = 1;
  size_t want = (vec_per_rank + kThreads * 2 - 1) / (kThreads * 2);   // >= 2 vectors per thread before adding CTAs
  if (want < 1) want = 1;
  if (want > (size_t)cap) want = cap;
  return (int)want;
}

// With two ranks the direct exchange moves S/2 per direction while the switch path moves 1.5 S.
bool prefer_nvls(const BnetColl* c) { return c->mc_ready && c->world > 2; }

}  // namespace

BNET_API const char* bnet_coll_last_error(void) { return g_err.c_str(); }

BNET_API int bnet_coll_create(int rank, int world, int dev, size_t heap_bytes, BnetColl** out) {
  if (world < 1 || world > BNET_COLL_MAX_WORLD || rank < 0 || rank >= world) return fail("bad rank/world %d/%d", rank, world);
  cudaError_t ce = cudaSetDevice(dev);
  if (ce != cudaSuccess) return fail("cudaSetDevice(%d): %s", dev, cudaGetErrorString(ce));
  cudaFree(0);   // make sure the primary context exists before driver-API calls
  const auto& d = driver();
  BnetColl* c = new BnetColl();
  c->rank = rank;
  c->world = world;
  c->dev = dev;
  c->heap_bytes = heap_bytes;
  void* sdev = nullptr;
  if (cudaHostAlloc((void**)&c->status_host, 64, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess ||
      cudaHostGetDevicePointer(&sdev, c->status_host, 0) != cudaSuccess) {
    delete c;
    return fail("cudaHostAlloc(status) failed");
  }
  *c->status_host = 0;
  c->status_dev = (uint32_t*)sdev;
  size_t want = kPadBytes + heap_bytes;
  if (!d.ok) {
    if (world > 1) { delete c; return fail("CUDA driver API unavailable: multi-GPU symmetric memory needs cuMem*"); }
    void* p = nullptr;
    if (cudaMalloc(&p, want) != cudaSuccess) { delete c; return fail("cudaMalloc(%zu) failed", want); }
    cudaMemset(p, 0, kPadBytes);
    c->local_va = (CUdeviceptr)p;
    c->alloc_bytes = want;
    c->vmm = false;
  } else {
    CUmemAllocationProp prop{};
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = dev;
    prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t gran = 2 << 20;
    d.MemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED);
    // multicast support + granularity
    int mc_attr = 0;
    CUdevice cudev;
    if (world > 1 && d.MulticastCreate && env_int("COLL_MULTICAST", 1) && d.DeviceGet(&cudev, dev) == CUDA_SUCCESS &&
        d.DeviceGetAttribute(&mc_attr, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, cudev) == CUDA_SUCCESS && mc_attr) {
      c->mc_supported = true;
      CUmulticastObjectProp mp{};
      mp.numDevices = (unsigned)world;
      mp.size = want;
      mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
      size_t mg = 0;
      if (d.MulticastGetGranularity(&mg, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && mg > gran) gran = mg;
    }
    c->alloc_bytes = (want + gran - 1) / gran * gran;
    CUresult r = d.MemCreate(&c->mem, c->alloc_bytes, &prop, 0);
    if (r != CUDA_SUCCESS) { delete c; return fail("cuMemCreate(%zu): %s", c->alloc_bytes, cu_err(r)); }
    if (map_handle(c->mem, c->alloc_bytes, dev, &c->local_va) != 0) { d.MemRelease(c->mem); delete c; return -1; }
    cudaMemset((void*)c->local_va, 0, kPadBytes);
    c->vmm = true;
    if (world > 1) {
      r = d.MemExportToShareableHandle(&c->mem_fd, c->mem, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
      if (r != CUDA_SUCCESS) { delete c; return fail("cuMemExportToShareableHandle: %s", cu_err(r)); }
    }
    if (c->mc_supported && rank == 0) {
      CUmulticastObjectProp mp{};
      mp.numDevices = (unsigned)world;
      mp.size = c->alloc_bytes;
      mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
      r = d.MulticastCreate(&c->mc, &mp);
      if (r == CUDA_SUCCESS) r = d.MemExportToShareableHandle(&c->mc_fd, c->mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
      if (r != CUDA_SUCCESS) {
        BNET_INFO("coll: cuMulticastCreate unavailable (%s): falling back to P2P kernels", cu_err(r));
        c->mc_supported = false;
        c->mc = 0;
      }
    }
  }
  cudaDeviceSynchronize();
  c->peer_va[rank] = c->local_va;
  *out = c;
  return 0;
}

BNET_API int bnet_coll_export(BnetColl* c, void* blob_out) {
  Blob b{};
  b.magic = 0x434f4c4cu;
  b.rank = c->rank;
  b.dev = c->dev;
  b.pid = (uint32_t)getpid();
  b.alloc_bytes = c->alloc_bytes;
  b.has_mc = (c->rank == 0 && c->mc_supported && c->mc_fd >= 0) ? 1 : 0;
  if (c->world > 1) {
    // one-shot fd server: every peer connects once and receives our heap fd (and the multicast fd from rank 0)
    char name[64];
    snprintf(name, sizeof(name), "bnet-coll-%d-%016llx", (int)getpid(), (unsigned long long)random_u64());
    c->uds_name = name;
    int fd = socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
    sockaddr_un un{};
    un.sun_family = AF_UNIX;
    memcpy(un.sun_path + 1, name, strlen(name));
    socklen_t len = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + strlen(name));
    if (fd < 0 || bind(fd, (sockaddr*)&un, len) != 0 || listen(fd, 64) != 0) return fail("fd server: %s", strerror(errno));
    c->srv_fd = fd;
    snprintf(b.uds, sizeof(b.uds), "%s", name);
    int nclients = c->world - 1;
    int heap_fd = c->mem_fd, mc_fd = b.has_mc ? c->mc_fd : -1;
    c->srv = std::thread([fd, nclients, heap_fd, mc_fd] {
      for (int i = 0; i < nclients; i++) {
        pollfd p{fd, POLLIN, 0};
        if (poll(&p, 1, 120000) <= 0) break;
        int cfd = accept4(fd, nullptr, nullptr, SOCK_CLOEXEC);
        if (cfd < 0) break;
        send_fd_msg(cfd, 1, heap_fd);
        if (mc_fd >= 0) send_fd_msg(cfd, 2, mc_fd);
        close(cfd);
      }
    });
  }
  memset(blob_out, 0, BNET_COLL_BLOB_BYTES);
  memcpy(blob_out, &b, sizeof(b));
  return 0;
}

BNET_API int bnet_coll_import(BnetColl* c, const void* blobs) {
  const auto& d = driver();
  cudaSetDevice(c->dev);
  bool mc_exists = false;
  for (int p = 0; p < c->world; p++) {
    Blob b;
    memcpy(&b, (const char*)blobs + (size_t)p * BNET_COLL_BLOB_BYTES, sizeof(b));
    if (b.magic != 0x434f4c4cu || b.rank != p) return fail("bad blob for rank %d", p);
    if (b.alloc_bytes != c->alloc_bytes) return fail("rank %d allocated %llu bytes, we %zu", p, (unsigned long long)b.alloc_bytes, c->alloc_bytes);
    if (p == 0) mc_exists = b.has_mc != 0;
    if (p == c->rank) continue;
    int s = socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
    sockaddr_un un{};
    un.sun_family = AF_UNIX;
    memcpy(un.sun_path + 1, b.uds, strlen(b.uds));
    socklen_t len = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + strlen(b.uds));
    if (s < 0 || connect(s, (sockaddr*)&un, len) != 0) {
      if (s >= 0) close(s);
      return fail("connect to rank %d fd server: %s", p, strerror(errno));
    }
    uint32_t tag = 0;
    int fd = -1;
    if (recv_fd_msg(s, &tag, &fd) != 0 || tag != 1) { close(s); return fail("no heap fd from rank %d", p); }
    CUresult r = d.MemImportFromShareableHandle(&c->peer_mem[p], (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
    close(fd);
    if (r != CUDA_SUCCESS) { close(s); return fail("import heap of rank %d: %s", p, cu_err(r)); }
    if (map_handle(c->peer_mem[p], c->alloc_bytes, c->dev, &c->peer_va[p]) != 0) { close(s); return -1; }
    if (p == 0 && mc_exists) {
      int mfd = -1;
      if (recv_fd_msg(s, &tag, &mfd) == 0 && tag == 2) {
        r = d.MemImportFromShareableHandle(&c->mc, (void*)(uintptr_t)mfd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
        close(mfd);
        if (r != CUDA_SUCCESS) { BNET_INFO("coll: import multicast handle: %s", cu_err(r)); c->mc = 0; }
      }
    }
    close(s);
  }
  if (c->srv.joinable()) c->srv.join();
  if (c->srv_fd >= 0) { close(c->srv_fd); c->srv_fd = -1; }
  c->mc_supported = mc_exists && c->mc != 0;
  return 0;
}

BNET_API int bnet_coll_mc_add_device(BnetColl* c) {
  if (!c->mc_supported) return 0;
  const auto& d = driver();
  CUdevice cudev;
  d.DeviceGet(&cudev, c->dev);
  CUresult r = d.MulticastAddDevice(c->mc, cudev);
  if (r != CUDA_SUCCESS) {
    BNET_INFO("coll: cuMulticastAddDevice: %s -> P2P kernels", cu_err(r));
    c->mc_supported = false;
    return 1;   // caller must agree on the outcome across ranks
  }
  return 0;
}

BNET_API int bnet_coll_mc_bind(BnetColl* c) {
  if (!c->mc_supported) return 0;
  const auto& d = driver();
  CUresult r = d.MulticastBindMem(c->mc, 0, c->mem, 0, c->alloc_bytes, 0);
  if (r != CUDA_SUCCESS) {
    BNET_INFO("coll: cuMulticastBindMem: %s -> P2P kernels", cu_err(r));
    c->mc_supported = false;
    return 1;
  }
  if (map_handle(c->mc, c->alloc_bytes, c->dev, &c->mc_va) != 0) {
    c->mc_supported = false;
    return 1;
  }
  c->mc_ready = true;
  return 0;
}

static void refresh_devp(BnetColl* c) {
  CollDev& p = c->devp;
  for (int i = 0; i < BNET_COLL_MAX_WORLD; i++) p.heap[i] = i < c->world ? (char*)c->peer_va[i] : nullptr;
  p.mc = c->mc_ready ? (char*)c->mc_va : nullptr;
  p.status = c->status_dev;
  p.rank = c->rank;
  p.world = c->world;
}

BNET_API int bnet_coll_destroy(BnetColl* c) {
  if (!c) return 0;
  cudaSetDevice(c->dev);
  cudaDeviceSynchronize();
  const auto& d = driver();
  if (c->srv.joinable()) c->srv.join();
  if (c->vmm) {
    if (c->mc_va) { d.MemUnmap(c->mc_va, c->alloc_bytes); d.MemAddressFree(c->mc_va, c->alloc_bytes); }
    if (c->mc) {
      CUdevice cudev;
      d.DeviceGet(&cudev, c->dev);
      if (c->mc_ready) d.MulticastUnbind(c->mc, cudev, 0, c->alloc_bytes);
      d.MemRelease(c->mc);
    }
    for (int p = 0; p < c->world; p++) {
      if (p == c->rank || !c->peer_va[p]) continue;
      d.MemUnmap(c->peer_va[p], c->alloc_bytes);
      d.MemAddressFree(c->peer_va[p], c->alloc_bytes);
      d.MemRelease(c->peer_mem[p]);
    }
    d.MemUnmap(c->local_va, c->alloc_bytes);
    d.MemAddressFree(c->local_va, c->alloc_bytes);
    d.MemRelease(c->mem);
    if (c->mem_fd >= 0) close(c->mem_fd);
    if (c->mc_fd >= 0) close(c->mc_fd);
  } else if (c->local_va) {
    cudaFree((void*)c->local_va);
  }
  if (c->status_host) cudaFreeHost(c->status_host);
  delete c;
  return 0;
}

BNET_API void* bnet_coll_heap(BnetColl* c) { return (char*)c->local_va + kPadBytes; }
BNET_API size_t bnet_coll_heap_bytes(BnetColl* c) { return c->alloc_bytes - kPadBytes; }
BNET_API void* bnet_coll_peer_heap(BnetColl* c, int peer) {
  return (peer >= 0 && peer < c->world && c->peer_va[peer]) ? (char*)c->peer_va[peer] + kPadBytes : nullptr;
}
BNET_API void* bnet_coll_mc_heap(BnetColl* c) { return c->mc_ready ? (char*)c->mc_va + kPadBytes : nullptr; }
BNET_API int bnet_coll_has_multicast(BnetColl* c) { return c->mc_ready ? 1 : 0; }
BNET_API unsigned bnet_coll_status(BnetColl* c) { return *(volatile uint32_t*)c->status_host; }

// ---- dispatch helpers -------------------------------------------------------------------------
template <int DT, int OP>
static int run_allreduce(BnetColl* c, int algo, size_t off, size_t nvec, int chan, int nb, cudaStream_t st) {
  if (algo == BNET_ALGO_NVLS) return launch(bnet_allreduce_nvls_kernel<DT, OP>, nb, kThreads, st, c->devp, off, nvec, chan);
  return launch(bnet_allreduce_p2p_kernel<DT, OP>, nb, kThreads, st, c->devp, off, nvec, chan);
}

template <int DT>
static int run_allreduce_op(BnetColl* c, int op, int algo, size_t off, size_t nvec, int chan, int nb, cudaStream_t st) {
  switch (op) {
    case BNET_SUM: return run_allreduce<DT, BNET_SUM>(c, algo, off, nvec, chan, nb, st);
    case BNET_AVG: return run_allreduce<DT, BNET_AVG>(c, algo, off, nvec, chan, nb, st);
    case BNET_MAX:
      if constexpr (DT == BNET_F32) { if (algo == BNET_ALGO_NVLS) algo = BNET_ALGO_P2P_TWOSHOT; return launch(bnet_allreduce_p2p_kernel<DT, BNET_MAX>, nb, kThreads, st, c->devp, off, nvec, chan); }
      else return run_allreduce<DT, BNET_MAX>(c, algo, off, nvec, chan, nb, st);
    case BNET_MIN:
      if constexpr (DT == BNET_F32) { return launch(bnet_allreduce_p2p_kernel<DT, BNET_MIN>, nb, kThreads, st, c->devp, off, nvec, chan); }
      else return run_allreduce<DT, BNET_MIN>(c, algo, off, nvec, chan, nb, st);
  }
  return fail("bad op %d", op);
}

static size_t elsize(int dt) { return dt == BNET_F32 ? 4 : 2; }

BNET_API int bnet_allreduce(BnetColl* c, size_t offset, size_t count, int dtype, int op, int algo, int channel,
                            int nblocks, void* stream) {
  if (channel < 0 || channel >= BNET_COLL_CHANNELS) return fail("bad channel");
  size_t bytes = count * elsize(dtype);
  if (bytes % (16 * (size_t)c->world) || offset % 16) return fail("all-reduce needs offset%%16==0 and bytes%%(16*world)==0 (got %zu,%zu)", offset, bytes);
  if (offset + bytes > c->alloc_bytes - kPadBytes) return fail("all-reduce range outside the heap");
  refresh_devp(c);
  if (c->world == 1) return 0;   // nothing to reduce
  if (algo == BNET_ALGO_AUTO) algo = prefer_nvls(c) ? BNET_ALGO_NVLS : BNET_ALGO_P2P_TWOSHOT;
  if (algo == BNET_ALGO_NVLS && !c->mc_ready) return fail("NVLS requested but multicast is not available");
  size_t nvec = bytes / 16;
  int nb = pick_blocks(c, nvec / c->world, nblocks, algo == BNET_ALGO_NVLS ? BLK_NVLS : BLK_P2P);
  size_t off = kPadBytes + offset;
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case BNET_F32: return run_allreduce_op<BNET_F32>(c, op, algo, off, nvec, channel, nb, st);
    case BNET_BF16: return run_allreduce_op<BNET_BF16>(c, op, algo, off, nvec, channel, nb, st);
    case BNET_F16: return run_allreduce_op<BNET_F16>(c, op, algo, off, nvec, channel, nb, st);
  }
  return fail("bad dtype %d", dtype);
}

template <int DT>
static int run_oneshot(BnetColl* c, int op, size_t off, char* out, size_t nvec, int chan, int nb, cudaStream_t st) {
  switch (op) {
    case BNET_SUM: return launch(bnet_allreduce_oneshot_kernel<DT, BNET_SUM>, nb, kThreads, st, c->devp, off, out, nvec, chan);
    case BNET_AVG: return launch(bnet_allreduce_oneshot_kernel<DT, BNET_AVG>, nb, kThreads, st, c->devp, off, out, nvec, chan);
    case BNET_MAX: return launch(bnet_allreduce_oneshot_kernel<DT, BNET_MAX>, nb, kThreads, st, c->devp, off, out, nvec, chan);
    case BNET_MIN: return launch(bnet_allreduce_oneshot_kernel<DT, BNET_MIN>, nb, kThreads, st, c->devp, off, out, nvec, chan);
  }
  return fail("bad op %d", op);
}

BNET_API int bnet_allreduce_oneshot(BnetColl* c, size_t offset, void* out, size_t count, int dtype, int op, int channel,
                                    int nblocks, void* stream) {
  if (channel < 0 || channel >= BNET_COLL_CHANNELS) return fail("bad channel");
  size_t bytes = count * elsize(dtype);
  if (bytes % 16 || offset % 16 || ((uintptr_t)out & 15)) return fail("one-shot all-reduce needs 16-byte alignment");
  refresh_devp(c);
  size_t nvec = bytes / 16;
  int nb = pick_blocks(c, nvec, nblocks, BLK_P2P);
  size_t off = kPadBytes + offset;
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case BNET_F32: return run_oneshot<BNET_F32>(c, op, off, (char*)out, nvec, channel, nb, st);
    case BNET_BF16: return run_oneshot<BNET_BF16>(c, op, off, (char*)out, nvec, channel, nb, st);
    case BNET_F16: return run_oneshot<BNET_F16>(c, op, off, (char*)out, nvec, channel, nb, st);
  }
  return fail("bad dtype %d", dtype);
}

template <int DT>
static int run_ll(BnetColl* c, int op, size_t ll_off, size_t ll_words, const void* in, void* out, size_t nwords, size_t nelem,
                  cudaStream_t st) {
  const int nb = (int)((nwords + 255) / 256);
  const uint32_t* i32 = (const uint32_t*)in;
  uint32_t* o32 = (uint32_t*)out;
  switch (op) {
    case BNET_SUM: return launch(bnet_allreduce_ll_kernel<DT, BNET_SUM>, nb, 256, st, c->devp, ll_off, ll_words, i32, o32, nwords, nelem);
    case BNET_AVG: return launch(bnet_allreduce_ll_kernel<DT, BNET_AVG>, nb, 256, st, c->devp, ll_off, ll_words, i32, o32, nwords, nelem);
    case BNET_MAX: return launch(bnet_allreduce_ll_kernel<DT, BNET_MAX>, nb, 256, st, c->devp, ll_off, ll_words, i32, o32, nwords, nelem);
    case BNET_MIN: return launch(bnet_allreduce_ll_kernel<DT, BNET_MIN>, nb, 256, st, c->devp, ll_off, ll_words, i32, o32, nwords, nelem);
  }
  return fail("bad op %d", op);
}

// Small-message all-reduce without any barrier (see bnet_allreduce_ll_kernel).  `ll_offset`: byte offset in the heap of an
// area of 64 + 2 * world * ll_words * 8 bytes that is ZERO before the first call and used by nothing else; every rank makes
// the same sequence of calls on it.  in / out: local device pointers, 4-byte aligned, count elements.
BNET_API size_t bnet_allreduce_ll_area_bytes(int world, size_t ll_words) { return 64 + 2 * (size_t)world * ll_words * 8; }

BNET_API int bnet_allreduce_ll(BnetColl* c, size_t ll_offset, size_t ll_words, const void* in, void* out, size_t count, int dtype,
                               int op, void* stream) {
  const size_t es = elsize(dtype);
  const size_t nwords = (count * es + 3) / 4;
  if (nwords == 0) return 0;
  if (nwords > ll_words) return fail("message of %zu words does not fit the LL area (%zu words per sender)", nwords, ll_words);
  if (((uintptr_t)in & 3) || ((uintptr_t)out & 3) || (ll_offset & 7)) return fail("LL all-reduce needs 4-byte aligned buffers");
  if (ll_offset + bnet_allreduce_ll_area_bytes(c->world, ll_words) > c->heap_bytes) return fail("LL area outside the heap");
  refresh_devp(c);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t off = kPadBytes + ll_offset;
  switch (dtype) {
    case BNET_F32: return run_ll<BNET_F32>(c, op, off, ll_words, in, out, nwords, count, st);
    case BNET_BF16: return run_ll<BNET_BF16>(c, op, off, ll_words, in, out, nwords, count, st);
    case BNET_F16: return run_ll<BNET_F16>(c, op, off, ll_words, in, out, nwords, count, st);
  }
  return fail("bad dtype %d", dtype);
}

BNET_API int bnet_barrier(BnetColl* c, int channel, void* stream) {
  refresh_devp(c);
  if (c->world == 1) return 0;
  return launch(bnet_barrier_kernel, 1, kThreads, (cudaStream_t)stream, c->devp, channel);
}

template <int DT>
static int run_fused(BnetColl* c, size_t goff, size_t poff, size_t nvec, float lr, float mu, float wd, float gs,
                     float* master, float* mom, int zero, int chan, int nb, cudaStream_t st, const float* hp) {
  if (c->world == 1)
    return launch(bnet_fused_sgd_kernel<DT, 0>, nb, kThreads, st, c->devp, goff, poff, nvec, lr, mu, wd, gs, master, mom, zero, chan, hp);
  if (prefer_nvls(c) && env_int("FUSED_NVLS", 1))
    return launch(bnet_fused_sgd_kernel<DT, 1>, nb, kThreads, st, c->devp, goff, poff, nvec, lr, mu, wd, gs, master, mom, zero, chan, hp);
  return launch(bnet_fused_sgd_kernel<DT, 2>, nb, kThreads, st, c->devp, goff, poff, nvec, lr, mu, wd, gs, master, mom, zero, chan, hp);
}

static int fused_allreduce_sgd_impl(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype, float lr,
                                    float momentum, float weight_decay, float grad_scale, float* master, float* mom_buf,
                                    int zero_grads, int channel, int nblocks, void* stream, const float* hp);

BNET_API int bnet_fused_allreduce_sgd(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype, float lr,
                                      float momentum, float weight_decay, float grad_scale, float* master,
                                      float* mom_buf, int zero_grads, int channel, int nblocks, void* stream) {
  return fused_allreduce_sgd_impl(c, grad_off, param_off, count, dtype, lr, momentum, weight_decay, grad_scale, master, mom_buf,
                                  zero_grads, channel, nblocks, stream, nullptr);
}

// Same, with {lr, momentum, weight_decay, grad_scale} read from 4 floats of device memory at kernel run time.
BNET_API int bnet_fused_allreduce_sgd_hp(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype,
                                         const float* hp_dev, float* master, float* mom_buf, int zero_grads, int channel,
                                         int nblocks, void* stream) {
  if (!hp_dev || ((uintptr_t)hp_dev & 15)) return fail("hyper-parameter block must be a 16-byte aligned device pointer");
  return fused_allreduce_sgd_impl(c, grad_off, param_off, count, dtype, 0.f, 0.f, 0.f, 1.f, master, mom_buf, zero_grads, channel,
                                  nblocks, stream, hp_dev);
}

static int fused_allreduce_sgd_impl(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype, float lr,
                                    float momentum, float weight_decay, float grad_scale, float* master, float* mom_buf,
                                    int zero_grads, int channel, int nblocks, void* stream, const float* hp) {
  if (channel < 0 || channel >= BNET_COLL_CHANNELS) return fail("bad channel");
  if (dtype != BNET_F32 && dtype != BNET_BF16) return fail("fused SGD supports f32 and bf16");
  size_t bytes = count * elsize(dtype);
  if (bytes % (16 * (size_t)c->world) || grad_off % 16 || param_off % 16) return fail("fused SGD needs 16-byte aligned offsets and bytes%%(16*world)==0");
  if (grad_off + bytes > c->alloc_bytes - kPadBytes || param_off + bytes > c->alloc_bytes - kPadBytes) return fail("fused SGD range outside the heap");
  if (((uintptr_t)master | (uintptr_t)mom_buf) & 15) return fail("optimizer state must be 16-byte aligned");
  refresh_devp(c);
  size_t nvec = bytes / 16;
  int nb = pick_blocks(c, nvec / c->world, nblocks, prefer_nvls(c) && env_int("FUSED_NVLS", 1) ? BLK_FUSED_NVLS : BLK_P2P);
  cudaStream_t st = (cudaStream_t)stream;
  size_t goff = kPadBytes + grad_off, poff = kPadBytes + param_off;
  if (dtype == BNET_F32) return run_fused<BNET_F32>(c, goff, poff, nvec, lr, momentum, weight_decay, grad_scale, master, mom_buf, zero_grads, channel, nb, st, hp);
  return run_fused<BNET_BF16>(c, goff, poff, nvec, lr, momentum, weight_decay, grad_scale, master, mom_buf, zero_grads, channel, nb, st, hp);
}

BNET_API int bnet_pack_cast(const BnetPackItem* items_dev, int n, void* dst, int src_dtype, int dst_dtype, float scale,
                            uint64_t max_numel, void* stream) {
  if (n <= 0) return 0;
  int gx = (int)((max_numel + 256 * 8 - 1) / (256 * 8));
  if (gx < 1) gx = 1;
  if (gx > 64) gx = 64;
  dim3 grid(gx, n);
  cudaStream_t st = (cudaStream_t)stream;
  if (src_dtype == BNET_F32 && dst_dtype == BNET_BF16) bnet_pack_cast_kernel<float, __nv_bfloat16><<<grid, 256, 0, st>>>(items_dev, (__nv_bfloat16*)dst, scale);
  else if (src_dtype == BNET_BF16 && dst_dtype == BNET_BF16) bnet_pack_cast_kernel<__nv_bfloat16, __nv_bfloat16><<<grid, 256, 0, st>>>(items_dev, (__nv_bfloat16*)dst, scale);
  else if (src_dtype == BNET_BF16 && dst_dtype == BNET_F32) bnet_pack_cast_kernel<__nv_bfloat16, float><<<grid, 256, 0, st>>>(items_dev, (float*)dst, scale);
  else if (src_dtype == BNET_F32 && dst_dtype == BNET_F32) bnet_pack_cast_kernel<float, float><<<grid, 256, 0, st>>>(items_dev, (float*)dst, scale);
  else if (src_dtype == BNET_F16 && dst_dtype == BNET_F32) bnet_pack_cast_kernel<__half, float><<<grid, 256, 0, st>>>(items_dev, (float*)dst, scale);
  else return fail("unsupported pack/cast %d->%d", src_dtype, dst_dtype);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail("pack kernel launch failed: %s", cudaGetErrorString(e));
  return 1;
}

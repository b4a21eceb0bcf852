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
#include <type_traits>
#include <vector>

#include "bnet/bnet_coll.h"
#include "core/common.h"
#include "cuda/driver_api.h"
#include "cuda/optim_body.cuh"
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
// (add only: max and min take the peer-load kernel, see run_allreduce_op)
template <int DT, int OP>
__device__ __forceinline__ int4 mc_ld_reduce(const char* p) {
  static_assert(OP == BNET_SUM || OP == BNET_AVG, "the in-switch reduction is used for add only");
  int4 r;
  if constexpr (DT == BNET_F32) {
    float4 f = ptx::multimem_ld_reduce_add_f32x4(p);
    r.x = __float_as_int(f.x); r.y = __float_as_int(f.y); r.z = __float_as_int(f.z); r.w = __float_as_int(f.w);
  } else if constexpr (DT == BNET_BF16) {
    r = ptx::multimem_ld_reduce_add_bf16x8(p);
  } else {
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

// ------------------------------------------------------------------ fused all-reduce + optimizer + broadcast
// MODE 0: single GPU, 1: NVLS multicast, 2: peer loads/stores
//
// The summed gradient vector at heap byte offset `go` (MODE 1: in-switch reduction, raw vector in gv; MODE 2: peer
// loads summed in fp32 into gf; MODE 0: the local vector in gv) ...
template <int DT, int MODE>
__device__ __forceinline__ void fused_grad_issue(const CollDev& d, size_t go, int4& gv, float* gf) {
  if constexpr (MODE == 1) gv = mc_ld_reduce<DT, BNET_SUM>(d.mc + go);
  else if constexpr (MODE == 2) p2p_reduce<DT, BNET_SUM>(d, go, d.rank, gf);
  else gv = ptx::ld_na_v4(reinterpret_cast<const int4*>(d.heap[0] + go));
}
// ... as fp32 lanes.  For bf16 gradients the modes differ before the fp32 update: MODE 1 gets the switch's sum
// rounded to bf16 (the switch returns the dtype), MODE 2 keeps the fp32 sum of the peer loads.
template <int DT, int MODE>
__device__ __forceinline__ void fused_grad_get(const int4& gv, const float* gf, float* g) {
  if constexpr (MODE == 2) {
#pragma unroll
    for (int k = 0; k < VecTraits<DT>::kElems; k++) g[k] = gf[k];
  } else {
    unpack<DT>(gv, g);
  }
}
// ... and the new parameter vector `out` stored at heap byte offset `po` on every rank
template <int MODE>
__device__ __forceinline__ void fused_param_store(const CollDev& d, size_t po, const int4& out) {
  if constexpr (MODE == 1) {
    ptx::multimem_st_v4(d.mc + po, out);          // new parameters land on every rank
  } else if constexpr (MODE == 2) {
    for (int j = 0; j < d.world; j++) {
      int pr = d.rank + j;
      if (pr >= d.world) pr -= d.world;
      ptx::st_na_v4(reinterpret_cast<int4*>(d.heap[pr] + po), out);
    }
  } else {
    ptx::st_na_v4(reinterpret_cast<int4*>(d.heap[0] + po), out);
  }
}

// Reset our gradients for the next backward, after the closing rank_barrier.  The barrier only pairs CTA b with
// CTA b of the peers (CTAs of a grid start staggered when the kernel runs under backward on the side stream), so
// CTA b may only zero what CTA b of some rank has READ: shard p, vectors p*per + i for exactly the i this CTA walks
// in the update loop.  Zeroing with a flat index would hand vectors of shard p >= 1 to a different CTA than the one
// rank p reads them with.
__device__ __forceinline__ void fused_zero_grads(const CollDev& d, size_t goff, size_t nvec, size_t per, size_t stride) {
  int4* gz = reinterpret_cast<int4*>(d.heap[d.rank] + goff);
  const int4 z = make_int4(0, 0, 0, 0);
  for (int p = 0; p < d.world; p++)
    for (size_t j = (size_t)blockIdx.x * kThreads + threadIdx.x; j < per; j += stride) ptx::st_na_v4(gz + (size_t)p * per + j, z);
  // vectors beyond per*world are read by nobody
  for (size_t j = per * d.world + (size_t)blockIdx.x * kThreads + threadIdx.x; j < nvec; j += stride) ptx::st_na_v4(gz + j, z);
}

// Optimizer policies of the fused step: kStates fp32 arrays per element (master weights first), kU gradient vectors
// per thread per batch, and the per-element update of optim_body.cuh.
struct SgdOpt {
  static constexpr int kStates = 2;   // master, momentum
  static constexpr int kU = 2;        // (register budget: 2 CTAs/SM)
  float lr, mu, wd, gscale;
  __device__ __forceinline__ void update(float g, float (&s)[kStates][8], int k) const {
    optim::sgd_update(g, s[0][k], s[1][k], lr, mu, wd, gscale);
  }
};
// AdamW takes one vector per batch: two would hold 2*(3*E + 4) live values for bf16, and ptxas spills that at the
// 64-register cap of two 512-thread CTAs per SM.  One vector fits without spilling and still keeps
// 1024 threads * (16 + 12*E) bytes of loads in flight per SM.
struct AdamWOpt {
  static constexpr int kStates = 3;   // master, exp_avg, exp_avg_sq
  static constexpr int kU = 1;
  optim::AdamWCoef c;
  __device__ __forceinline__ void update(float g, float (&s)[kStates][8], int k) const {
    optim::adamw_update(g, s[0][k], s[1][k], s[2][k], c);
  }
};

// Where the fused step takes the rank-summed gradient from.  HeapGrad: the bucket's gradients at heap byte offset `off`,
// reduced over the ranks on the fly (fused_grad_issue / fused_grad_get).  ScratchGrad: this rank's shard of them,
// already reduced into local fp32 memory by bnet_clip_norm_kernel (the same floats fused_grad_get would give), times
// the clipping coefficient.
struct HeapGrad {
  size_t off;
};
struct ScratchGrad {
  const float* g;
  float coef;
};
// LARS: the scratch as in ScratchGrad, but every vector scaled by its own tensor's gradient scale (which folds in the
// clipping coefficient and the trust ratio) and decayed by its tensor's weight decay: the pair scal[tensor], where the
// tensor is the one of the segment (BnetLarsSeg, sorted by vec0) that holds the shard vector.
struct LarsGrad {
  const float* g;
  const int4* seg;   // {vec0, nvec, tensor, slot0}
  int nseg;
  const float2* scal;
};
// The update scalars of shard vector v's tensor, found by a binary search over the sorted segment starts, in L1-resident table entries.
__device__ __forceinline__ float2 lars_vec_scalars(const LarsGrad& s, size_t v) {
  int lo = 0, hi = s.nseg - 1;
  while (lo < hi) {
    const int m = (lo + hi + 1) >> 1;
    if ((size_t)__ldg(&s.seg[m].x) <= v) lo = m;
    else hi = m - 1;
  }
  return __ldg(s.scal + __ldg(&s.seg[lo].z));
}
// SGD with momentum whose gradient scale and weight decay come per vector from LarsGrad (lr and momentum are the step's).
// U vectors per batch: the bf16 variants take one, as AdamW does, because the table search on top of two vectors'
// loads spills at the 64-register cap of two 512-thread CTAs per SM.
template <int U>
struct LarsOpt {
  static constexpr int kStates = 2;   // master, momentum
  static constexpr int kU = U;
  float lr, mu;
};

// Parameter groups: the step of SgdOpt / AdamWOpt with every vector's group's scalars.  `at(v)` finds shard vector v's
// group in the sorted segment table with a per-thread cursor (optim::group_seg_advance; v only increases within a
// thread) and returns the ungrouped policy with that group's values, from shared memory.  The cursor starts at the
// thread's first vector.
struct GroupSegs {
  const int* seg;   // BnetGroupSeg rows, 4 ints each
  int nseg;
  mutable int cur;
  __device__ __forceinline__ GroupSegs(const int4* s, int n)
      : seg(reinterpret_cast<const int*>(s)), nseg(n), cur(optim::group_seg_find(seg, n, (int)(blockIdx.x * kThreads + threadIdx.x))) {}
  __device__ __forceinline__ int group(size_t v) const {
    cur = optim::group_seg_advance(seg, nseg, cur, (int)v);
    return __ldg(seg + 4 * cur + 2);
  }
};
// SGD: {lr, weight decay} per group in shared memory; momentum and gradient scale are the step's.  U vectors per batch.
template <int U>
struct SgdGroupsOpt {
  static constexpr int kStates = 2;   // master, momentum
  static constexpr int kU = U;
  float mu, gscale;
  const float2* grp;
  GroupSegs segs;
  __device__ __forceinline__ SgdOpt at(size_t v) const {
    const float2 s = grp[segs.group(v)];
    return SgdOpt{s.x, mu, s.y, gscale};
  }
};
// AdamW: every group's coefficients, computed once per CTA into shared memory.  Only decay and step_size depend on the
// group's lr and weight decay; the others are the same in every row and stay in registers (`c`, group 0's row), so a
// vector reads two floats.  (Copying a whole row per vector spills the bf16 variants.)  One vector per batch, as AdamWOpt.
struct AdamWGroupsOpt {
  static constexpr int kStates = 3;   // master, exp_avg, exp_avg_sq
  static constexpr int kU = 1;
  optim::AdamWCoef c;
  const optim::AdamWCoef* coef;
  GroupSegs segs;
  __device__ __forceinline__ AdamWOpt at(size_t v) const {
    const optim::AdamWCoef& r = coef[segs.group(v)];
    AdamWOpt o{c};
    o.c.decay = r.decay;
    o.c.step_size = r.step_size;
    return o;
  }
};
template <class Opt> constexpr bool kGroupedOpt = false;
template <int U> constexpr bool kGroupedOpt<SgdGroupsOpt<U>> = true;
template <> constexpr bool kGroupedOpt<AdamWGroupsOpt> = true;

// One batch = U 16-byte gradient vectors per thread.  All loads of the batch (in-switch reductions / peer loads or the
// fp32 scratch, the fp32 state) are issued before any dependent math so that U*(1 + S*E/4) requests per thread are in
// flight: the kernel is latency*bandwidth bound (NVLink round trip ~3 us, HBM), not ALU bound.
template <int DT, int MODE, int U, class Opt, class G>
__device__ __forceinline__ void fused_batch(const CollDev& d, const G& src, size_t poff, size_t start, size_t i, size_t stride,
                                            const Opt& opt, float* const (&state)[Opt::kStates]) {
  constexpr int E = VecTraits<DT>::kElems;
  constexpr int Q = E / 4;
  constexpr int S = Opt::kStates;
  constexpr bool kHeap = std::is_same<G, HeapGrad>::value;
  constexpr bool kLars = std::is_same<G, LarsGrad>::value;
  int4 gv[U];
  float4 sm[U][S][Q];
  float gp2p[(MODE == 2) ? U : 1][8];
  float4 gs[kHeap ? 1 : U][Q];
#pragma unroll
  for (int u = 0; u < U; u++) {
    if constexpr (kHeap) {
      fused_grad_issue<DT, MODE>(d, src.off + (start + i + u * stride) * 16, gv[u], gp2p[(MODE == 2) ? u : 0]);
    } else {
#pragma unroll
      for (int q = 0; q < Q; q++) gs[u][q] = ptx::ld_na_f4(reinterpret_cast<const float4*>(src.g + (i + u * stride) * E) + q);
    }
  }
#pragma unroll
  for (int u = 0; u < U; u++)
#pragma unroll
    for (int q = 0; q < Q; q++)
#pragma unroll
      for (int s = 0; s < S; s++) sm[u][s][q] = ptx::ld_na_f4(reinterpret_cast<const float4*>(state[s] + (i + u * stride) * E) + q);
#pragma unroll
  for (int u = 0; u < U; u++) {
    float g[8], st[S][8];
    [[maybe_unused]] float2 sc;
    if constexpr (kHeap) {
      fused_grad_get<DT, MODE>(gv[u], gp2p[(MODE == 2) ? u : 0], g);
    } else if constexpr (kLars) {
      // (the table search runs while the batch's later loads are still in flight)
      sc = lars_vec_scalars(src, i + u * stride);
#pragma unroll
      for (int q = 0; q < Q; q++) {
        g[4 * q] = gs[u][q].x * sc.x; g[4 * q + 1] = gs[u][q].y * sc.x;
        g[4 * q + 2] = gs[u][q].z * sc.x; g[4 * q + 3] = gs[u][q].w * sc.x;
      }
    } else {
#pragma unroll
      for (int q = 0; q < Q; q++) {
        g[4 * q] = gs[u][q].x * src.coef; g[4 * q + 1] = gs[u][q].y * src.coef;
        g[4 * q + 2] = gs[u][q].z * src.coef; g[4 * q + 3] = gs[u][q].w * src.coef;
      }
    }
#pragma unroll
    for (int q = 0; q < Q; q++)
#pragma unroll
      for (int s = 0; s < S; s++) {
        st[s][4 * q] = sm[u][s][q].x; st[s][4 * q + 1] = sm[u][s][q].y; st[s][4 * q + 2] = sm[u][s][q].z; st[s][4 * q + 3] = sm[u][s][q].w;
      }
    if constexpr (kLars) {
      // per-element sgd_update with the vector's scalars: g already carries its gradient scale
      const SgdOpt o{opt.lr, opt.mu, sc.y, 1.0f};
#pragma unroll
      for (int k = 0; k < E; k++) o.update(g[k], st, k);
    } else if constexpr (kGroupedOpt<Opt>) {
      const auto o = opt.at(i + u * stride);
#pragma unroll
      for (int k = 0; k < E; k++) o.update(g[k], st, k);
    } else {
#pragma unroll
      for (int k = 0; k < E; k++) opt.update(g[k], st, k);
    }
#pragma unroll
    for (int q = 0; q < Q; q++)
#pragma unroll
      for (int s = 0; s < S; s++)
        ptx::st_na_f4(reinterpret_cast<float4*>(state[s] + (i + u * stride) * E) + q,
                      make_float4(st[s][4 * q], st[s][4 * q + 1], st[s][4 * q + 2], st[s][4 * q + 3]));
    fused_param_store<MODE>(d, poff + (start + i + u * stride) * 16, pack<DT>(st[0]));
  }
}

// barrier, reduce + update + broadcast of this rank's shard, barrier, gradient zeroing.
// From the scratch (the clipped step's apply stage) there is neither the opening barrier nor the zeroing.  The opening
// barrier guards two things: every rank's gradients of the bucket are complete before peers read them, and no rank
// still reads its parameters (backward) when the new ones arrive.  The apply stage reads no peer's gradients, and it
// runs behind bnet_clip_coef_kernel, whose rank barrier every rank reaches only after its comm stream waited for its
// whole backward.  The gradients were zeroed by the norm stage.
template <int DT, int MODE, class Opt, class G>
__device__ __forceinline__ void fused_step(const CollDev& d, const G& src, size_t poff, size_t nvec, const Opt& opt,
                                           float* const (&state)[Opt::kStates], int zero_grads, int chan) {
  constexpr bool kHeap = std::is_same<G, HeapGrad>::value;
  if constexpr (MODE != 0 && kHeap) rank_barrier(d, chan);
  const size_t per = nvec / d.world;
  const size_t start = (size_t)d.rank * per;
  const size_t stride = (size_t)gridDim.x * kThreads;
  constexpr int U = Opt::kU;
  size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
  for (; i + (U - 1) * stride < per; i += U * stride) fused_batch<DT, MODE, U>(d, src, poff, start, i, stride, opt, state);
  if constexpr (U > 1)
    for (; i < per; i += stride) fused_batch<DT, MODE, 1>(d, src, poff, start, i, stride, opt, state);
  if constexpr (MODE != 0) rank_barrier(d, chan);
  if constexpr (kHeap)
    if (zero_grads) fused_zero_grads(d, src.off, nvec, per, stride);
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
  float* const state[2] = {master, mom};
  fused_step<DT, MODE>(d, HeapGrad{goff}, poff, nvec, SgdOpt{lr, mu, wd, gscale}, state, zero_grads, chan);
}

// hp: the 8-float block of optim_body.cuh, always read from device memory.
template <int DT, int MODE>
__global__ void __launch_bounds__(kThreads, 2) bnet_fused_adamw_kernel(CollDev d, size_t goff, size_t poff, size_t nvec,
                                                                   const float* __restrict__ hp, float* __restrict__ master,
                                                                   float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                                                                   int zero_grads, int chan) {
  float* const state[3] = {master, exp_avg, exp_avg_sq};
  fused_step<DT, MODE>(d, HeapGrad{goff}, poff, nvec, AdamWOpt{optim::adamw_coef(hp)}, state, zero_grads, chan);
}

// ------------------------------------------------------------------ gradient clipping by global norm (three stages)
// Sum of one double per thread of a kThreads-thread CTA in a fixed order (a butterfly inside each warp, then the warps
// in order), so the same inputs give the same bits.  The sum is valid in thread 0.  One call per kernel.
__device__ __forceinline__ double cta_sum(double v) {
  __shared__ double warp_sums[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kThreads / 32; w++) s += warp_sums[w];
  return s;
}

// Stage 1, one launch per bucket from the gradient hook: barrier, reduce this rank's shard (the one-kernel path's
// fused_grad_issue / fused_grad_get), store the rank-summed gradient as fp32 into the local `scratch` shard, barrier,
// zero the gradients (the CTA-paired rule of fused_zero_grads).  Each CTA writes the sum of squares of what it stored
// to its own slot of the bucket's `partial` row (BNET_COLL_MAX_BLOCKS doubles; CTA 0 zeroes the slots beyond the
// grid).  No atomics: the same grid gives the same bits.  Squares and sums are taken in double: a square of an fp32
// value is exact there, and a sum of n of them is within n * 2^-53 of the exact one.
//
// ACC (gradient accumulation, every micro-batch after a bucket's first in the step): add the rank-summed gradient to
// what `scratch` already holds (scratch + g, in fp32) instead of storing it, and take the sums of squares over the new
// scratch values, so the bucket's partial row always describes its accumulated gradient.  The scratch loads are issued
// together with the gradient loads, before any dependent math, as fused_batch does; they go first because with peer
// loads (MODE 2) fused_grad_issue already sums, and in this order the bf16 P2P variant fits 64 registers unspilled.
template <int DT, int MODE, bool ACC>
__device__ __forceinline__ void reduce_norm_body(const CollDev& d, size_t goff, size_t nvec, float* __restrict__ scratch,
                                                 double* __restrict__ partial, int chan) {
  constexpr int E = VecTraits<DT>::kElems;
  constexpr int Q = E / 4;
  constexpr int U = 2;
  if constexpr (MODE != 0) rank_barrier(d, chan);
  const size_t per = nvec / d.world;
  const size_t start = (size_t)d.rank * per;
  const size_t stride = (size_t)gridDim.x * kThreads;
  double acc = 0.0;
  for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < per; i += U * stride) {
    int4 gv[U];
    float gp2p[(MODE == 2) ? U : 1][8];
    float4 sv[ACC ? U : 1][Q];
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (i + u * stride >= per) continue;
      if constexpr (ACC) {
#pragma unroll
        for (int q = 0; q < Q; q++) sv[u][q] = ptx::ld_na_f4(reinterpret_cast<const float4*>(scratch + (i + u * stride) * E) + q);
      }
      fused_grad_issue<DT, MODE>(d, goff + (start + i + u * stride) * 16, gv[u], gp2p[(MODE == 2) ? u : 0]);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (i + u * stride >= per) continue;
      float g[8];
      fused_grad_get<DT, MODE>(gv[u], gp2p[(MODE == 2) ? u : 0], g);
      if constexpr (ACC) {
#pragma unroll
        for (int q = 0; q < Q; q++) {
          g[4 * q] = sv[u][q].x + g[4 * q]; g[4 * q + 1] = sv[u][q].y + g[4 * q + 1];
          g[4 * q + 2] = sv[u][q].z + g[4 * q + 2]; g[4 * q + 3] = sv[u][q].w + g[4 * q + 3];
        }
      }
#pragma unroll
      for (int q = 0; q < Q; q++)
        ptx::st_na_f4(reinterpret_cast<float4*>(scratch + (i + u * stride) * E) + q,
                      make_float4(g[4 * q], g[4 * q + 1], g[4 * q + 2], g[4 * q + 3]));
#pragma unroll
      for (int k = 0; k < E; k++) acc = fma((double)g[k], (double)g[k], acc);
    }
  }
  acc = cta_sum(acc);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc;
  if (blockIdx.x == 0)
    for (int j = gridDim.x + threadIdx.x; j < BNET_COLL_MAX_BLOCKS; j += kThreads) partial[j] = 0.0;
  if constexpr (MODE != 0) rank_barrier(d, chan);
  fused_zero_grads(d, goff, nvec, per, stride);
}

template <int DT, int MODE>
__global__ void __launch_bounds__(kThreads, 2) bnet_clip_norm_kernel(CollDev d, size_t goff, size_t nvec, float* __restrict__ scratch,
                                                                 double* __restrict__ partial, int chan) {
  reduce_norm_body<DT, MODE, false>(d, goff, nvec, scratch, partial, chan);
}

// Stage 1 of an accumulating micro-batch: scratch += the rank-summed gradient (reduce_norm_body with ACC).
template <int DT, int MODE>
__global__ void __launch_bounds__(kThreads, 2) bnet_accum_norm_kernel(CollDev d, size_t goff, size_t nvec, float* __restrict__ scratch,
                                                                  double* __restrict__ partial, int chan) {
  reduce_norm_body<DT, MODE, true>(d, goff, nvec, scratch, partial, chan);
}

// Stage 2, one CTA per step after the last bucket's stage 1: sum this rank's `n` partials (all its rows) in a fixed
// order, exchange the per-rank sums through `world` doubles at heap byte offset `xoff`, add them in rank order
// 0..world-1 (every rank gets the same bits), and write total_norm = sqrt(sum) * gscale and clip_coef into the clip
// block.  The exchange slots are reused every step: the second rank barrier is passed only once every rank has read
// its slots, so no rank's next write can overtake a peer's read.
__global__ void __launch_bounds__(kThreads) bnet_clip_coef_kernel(CollDev d, const double* __restrict__ partials, size_t n,
                                                                 size_t xoff, float gscale, float* __restrict__ clip, int chan) {
  double s = 0.0;
  for (size_t j = threadIdx.x; j < n; j += kThreads) s += partials[j];
  s = cta_sum(s);
  if (d.world > 1) {
    if (threadIdx.x == 0)
      for (int p = 0; p < d.world; p++) reinterpret_cast<volatile double*>(d.heap[p] + xoff)[d.rank] = s;
    rank_barrier(d, chan);
    if (threadIdx.x == 0) {
      const volatile double* x = reinterpret_cast<const volatile double*>(d.heap[d.rank] + xoff);
      s = x[0];
      for (int q = 1; q < d.world; q++) s += x[q];
    }
    rank_barrier(d, chan);
  }
  if (threadIdx.x == 0) {
    const float total = (float)(sqrt(s) * (double)gscale);
    clip[optim::kClipTotalNorm] = total;
    clip[optim::kClipCoef] = optim::clip_coef(clip[optim::kClipMaxNorm], total);
  }
}

// Stage 3, one launch per bucket after stage 2: the optimizer step of fused_step from the fp32 scratch times clip_coef,
// then the parameter broadcast and the closing barrier.  Same hyper-parameters as bnet_fused_sgd_kernel /
// bnet_fused_adamw_kernel.
template <int DT, int MODE>
__global__ void __launch_bounds__(kThreads, 2) bnet_clip_apply_sgd_kernel(CollDev d, size_t poff, size_t nvec,
                                                                      const float* __restrict__ scratch, const float* __restrict__ clip,
                                                                      float lr, float mu, float wd, float gscale,
                                                                      float* __restrict__ master, float* __restrict__ mom, int chan,
                                                                      const float* __restrict__ hp) {
  if (hp != nullptr) {
    lr = hp[0];
    mu = hp[1];
    wd = hp[2];
    gscale = hp[3];
  }
  float* const state[2] = {master, mom};
  fused_step<DT, MODE>(d, ScratchGrad{scratch, clip[optim::kClipCoef]}, poff, nvec, SgdOpt{lr, mu, wd, gscale}, state, 0, chan);
}

template <int DT, int MODE>
__global__ void __launch_bounds__(kThreads, 2) bnet_clip_apply_adamw_kernel(CollDev d, size_t poff, size_t nvec,
                                                                        const float* __restrict__ scratch, const float* __restrict__ clip,
                                                                        const float* __restrict__ hp, float* __restrict__ master,
                                                                        float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                                                                        int chan) {
  float* const state[3] = {master, exp_avg, exp_avg_sq};
  fused_step<DT, MODE>(d, ScratchGrad{scratch, clip[optim::kClipCoef]}, poff, nvec, AdamWOpt{optim::adamw_coef(hp)}, state, 0,
                       chan);
}

// ------------------------------------------------------------------ parameter groups: per-group lr and weight decay
// The one-kernel steps (HeapGrad) and the staged step's apply stage (ScratchGrad) of SGD and AdamW with each vector's
// group's lr and weight decay from the group table (rows of optim::kGroupWords floats), found through the bucket's
// segment table.  Everything else -- barriers, gradient zeroing, parameter broadcast -- is fused_step's, unchanged.
//
// SGD: the first ngroups threads copy {lr, weight decay} of every group into shared memory; momentum and gradient
// scale come from the 4-float SGD block, whose lr and weight decay are not read.
__device__ __forceinline__ void sgd_groups_load(const float4* __restrict__ groups, int ngroups, float2* grp) {
  if ((int)threadIdx.x < ngroups) {
    const float4 r = groups[threadIdx.x];
    grp[threadIdx.x] = make_float2(r.x, r.y);
  }
  __syncthreads();
}
// AdamW: the first ngroups threads compute every group's coefficients with the unchanged optim::adamw_coef on a copy of
// the 8-float block with the group's lr and weight decay, so a group's elements get the bits of the ungrouped kernel
// run with those two values.  Before the opening rank barrier, where the wait for the peers hides it.
__device__ __forceinline__ void adamw_groups_coef(const float* __restrict__ hp, const float4* __restrict__ groups, int ngroups,
                                                  optim::AdamWCoef* coef) {
  if ((int)threadIdx.x < ngroups) {
    float h[optim::kHpWords];
#pragma unroll
    for (int k = 0; k < optim::kHpWords; k++) h[k] = hp[k];
    const float4 r = groups[threadIdx.x];
    h[optim::kHpLr] = r.x;
    h[optim::kHpWeightDecay] = r.y;
    coef[threadIdx.x] = optim::adamw_coef(h);
  }
  __syncthreads();
}
// Vectors per batch of the grouped SGD kernels: two, as SgdOpt, except in the bf16 apply stage, where the lookup on top
// of two vectors' scratch and state loads spills at the 64-register cap of two 512-thread CTAs per SM (as LarsOpt).

template <int DT, int MODE>
__global__ void __launch_bounds__(kThreads, 2) bnet_fused_sgd_groups_kernel(CollDev d, size_t goff, size_t poff, size_t nvec,
                                                                        const float* __restrict__ hp, const float4* __restrict__ groups,
                                                                        int ngroups, const int4* __restrict__ seg, int nseg,
                                                                        float* __restrict__ master, float* __restrict__ mom,
                                                                        int zero_grads, int chan) {
  __shared__ float2 grp[BNET_GROUPS_MAX];
  sgd_groups_load(groups, ngroups, grp);
  float* const state[2] = {master, mom};
  fused_step<DT, MODE>(d, HeapGrad{goff}, poff, nvec, SgdGroupsOpt<2>{hp[1], hp[3], grp, GroupSegs(seg, nseg)}, state,
                       zero_grads, chan);
}

template <int DT, int MODE>
__global__ void __launch_bounds__(kThreads, 2) bnet_fused_adamw_groups_kernel(CollDev d, size_t goff, size_t poff, size_t nvec,
                                                                          const float* __restrict__ hp, const float4* __restrict__ groups,
                                                                          int ngroups, const int4* __restrict__ seg, int nseg,
                                                                          float* __restrict__ master, float* __restrict__ exp_avg,
                                                                          float* __restrict__ exp_avg_sq, int zero_grads, int chan) {
  __shared__ optim::AdamWCoef coef[BNET_GROUPS_MAX];
  adamw_groups_coef(hp, groups, ngroups, coef);
  float* const state[3] = {master, exp_avg, exp_avg_sq};
  fused_step<DT, MODE>(d, HeapGrad{goff}, poff, nvec, AdamWGroupsOpt{coef[0], coef, GroupSegs(seg, nseg)}, state, zero_grads, chan);
}

template <int DT, int MODE>
__global__ void __launch_bounds__(kThreads, 2) bnet_clip_apply_sgd_groups_kernel(CollDev d, size_t poff, size_t nvec,
                                                                             const float* __restrict__ scratch, const float* __restrict__ clip,
                                                                             const float* __restrict__ hp, const float4* __restrict__ groups,
                                                                             int ngroups, const int4* __restrict__ seg, int nseg,
                                                                             float* __restrict__ master, float* __restrict__ mom, int chan) {
  __shared__ float2 grp[BNET_GROUPS_MAX];
  sgd_groups_load(groups, ngroups, grp);
  float* const state[2] = {master, mom};
  fused_step<DT, MODE>(d, ScratchGrad{scratch, clip[optim::kClipCoef]}, poff, nvec,
                       SgdGroupsOpt<DT == BNET_BF16 ? 1 : 2>{hp[1], hp[3], grp, GroupSegs(seg, nseg)}, state, 0, chan);
}

template <int DT, int MODE>
__global__ void __launch_bounds__(kThreads, 2) bnet_clip_apply_adamw_groups_kernel(CollDev d, size_t poff, size_t nvec,
                                                                               const float* __restrict__ scratch, const float* __restrict__ clip,
                                                                               const float* __restrict__ hp, const float4* __restrict__ groups,
                                                                               int ngroups, const int4* __restrict__ seg, int nseg,
                                                                               float* __restrict__ master, float* __restrict__ exp_avg,
                                                                               float* __restrict__ exp_avg_sq, int chan) {
  __shared__ optim::AdamWCoef coef[BNET_GROUPS_MAX];
  adamw_groups_coef(hp, groups, ngroups, coef);
  float* const state[3] = {master, exp_avg, exp_avg_sq};
  fused_step<DT, MODE>(d, ScratchGrad{scratch, clip[optim::kClipCoef]}, poff, nvec, AdamWGroupsOpt{coef[0], coef, GroupSegs(seg, nseg)}, state,
                       0, chan);
}

// ------------------------------------------------------------------ LARS: per-tensor trust ratios in the staged step
// Sums of two doubles per thread over a kThreads-thread CTA in a fixed order (cta_sum's butterfly, then the warps in
// order), valid in thread 0.  Unlike cta_sum it may be called repeatedly: the leading barrier keeps a call's writes of
// the warp sums behind the previous call's reads.
__device__ __forceinline__ double2 cta_sum2(double a, double b) {
  __shared__ double2 warp_sums[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = make_double2(a, b);
  __syncthreads();
  double2 s = make_double2(0.0, 0.0);
  if (threadIdx.x == 0)
    for (int w = 0; w < kThreads / 32; w++) {
      s.x += warp_sums[w].x;
      s.y += warp_sums[w].y;
    }
  return s;
}

// Per bucket, after stage 1: the sums of squares of this rank's fp32 master and scratch shards per chunk of
// BNET_LARS_CHUNK vectors of each segment, into the chunk's slot {sum w^2, sum g^2}.  A CTA takes whole chunks (grid
// stride over the bucket's `nslots` slots) and finds a slot's segment by a binary search over the segments' slot0.  Each
// chunk is summed the same way whichever CTA takes it, so the bits depend neither on the grid nor on a repeat, and no
// atomics are needed.  `q`: float4s per vector (1 for fp32 parameters, 2 for bf16).
__global__ void __launch_bounds__(kThreads) bnet_lars_norm_kernel(const float4* __restrict__ master, const float4* __restrict__ scratch,
                                                                 const int4* __restrict__ seg, int nseg, int q,
                                                                 double2* __restrict__ slots, int nslots) {
  for (int j = blockIdx.x; j < nslots; j += gridDim.x) {
    int lo = 0, hi = nseg - 1;
    while (lo < hi) {
      const int m = (lo + hi + 1) >> 1;
      if (__ldg(&seg[m].w) <= j) lo = m;
      else hi = m - 1;
    }
    const int4 s = __ldg(seg + lo);
    const size_t v0 = (size_t)s.x + (size_t)(j - s.w) * BNET_LARS_CHUNK;
    const size_t v1 = (size_t)s.x + (size_t)s.y < v0 + BNET_LARS_CHUNK ? (size_t)s.x + (size_t)s.y : v0 + BNET_LARS_CHUNK;
    double w2 = 0.0, g2 = 0.0;
#pragma unroll 4
    for (size_t f = v0 * q + threadIdx.x; f < v1 * q; f += kThreads) {
      const float4 w = ptx::ld_na_f4(master + f);
      const float4 g = ptx::ld_na_f4(scratch + f);
      w2 = fma((double)w.x, (double)w.x, w2); w2 = fma((double)w.y, (double)w.y, w2);
      w2 = fma((double)w.z, (double)w.z, w2); w2 = fma((double)w.w, (double)w.w, w2);
      g2 = fma((double)g.x, (double)g.x, g2); g2 = fma((double)g.y, (double)g.y, g2);
      g2 = fma((double)g.z, (double)g.z, g2); g2 = fma((double)g.w, (double)g.w, g2);
    }
    const double2 r = cta_sum2(w2, g2);
    if (threadIdx.x == 0) slots[j] = r;
  }
}

// Once per step, one CTA, after every bucket's norm launch: per tensor (one warp each, lanes over its slots, then a
// fixed butterfly) this rank's {sum w^2, sum g^2}, written into every rank's exchange area ([world][2][ntensors] doubles
// at heap byte offset `xoff`); after a rank barrier, per tensor (one thread each) the sums over the ranks in rank order
// 0..world-1 -- the same bits on every rank -- and the trust ratio and update scalars.  The second rank barrier lets the
// exchange area be reused next step, as in bnet_clip_coef_kernel; with one rank a CTA barrier stands for the first.
// Without clipping, the first barrier is the staged step's barrier before its update stage.
__global__ void __launch_bounds__(kThreads) bnet_lars_trust_kernel(CollDev d, const double2* __restrict__ slots,
                                                                  const int4* __restrict__ tens, int ntensors, size_t xoff,
                                                                  const float* __restrict__ clip, const float* __restrict__ hp,
                                                                  float2* __restrict__ scal, float* __restrict__ trust, int chan) {
  const int lane = threadIdx.x & 31;
  const size_t T = (size_t)ntensors;
  for (int j = threadIdx.x >> 5; j < ntensors; j += kThreads / 32) {
    const int4 t = tens[j];
    double w2 = 0.0, g2 = 0.0;
    for (int k = lane; k < t.y; k += 32) {
      const double2 s = slots[t.x + k];
      w2 += s.x;
      g2 += s.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      w2 += __shfl_xor_sync(0xffffffffu, w2, o);
      g2 += __shfl_xor_sync(0xffffffffu, g2, o);
    }
    if (lane == 0)
      for (int p = 0; p < d.world; p++) {
        volatile double* x = reinterpret_cast<volatile double*>(d.heap[p] + xoff) + 2 * T * d.rank;
        x[j] = w2;
        x[T + j] = g2;
      }
  }
  if (d.world > 1) {
    __threadfence_system();
    rank_barrier(d, chan);
  } else {
    __syncthreads();
  }
  const float coef = clip[optim::kClipCoef];
  const float gscale = hp[optim::kLarsGradScale], wd = hp[optim::kLarsWeightDecay];
  const float eta = hp[optim::kLarsEta], eps = hp[optim::kLarsEps];
  const float gs = gscale * coef;
  const volatile double* x = reinterpret_cast<const volatile double*>(d.heap[d.rank] + xoff);
  for (int j = threadIdx.x; j < ntensors; j += kThreads) {
    double w2 = x[j], g2 = x[T + j];
    for (int p = 1; p < d.world; p++) {
      w2 += x[2 * T * p + j];
      g2 += x[2 * T * p + T + j];
    }
    const float wn = (float)sqrt(w2);
    const float gn = (float)(sqrt(g2) * (double)gscale * (double)coef);
    const optim::LarsScalars ls = optim::lars_scalars(eta, eps, wd, gs, wn, gn, tens[j].z != 0);
    scal[j] = make_float2(ls.gscale, ls.wd);
    trust[j] = ls.t;
  }
  if (d.world > 1) rank_barrier(d, chan);
}

// Per bucket, after the trust kernel: fused_step from the scratch with each vector's tensor's scalars (LarsGrad), then
// the parameter broadcast and the closing barrier, as bnet_clip_apply_sgd_kernel.
template <int DT, int MODE>
__global__ void __launch_bounds__(kThreads, 2) bnet_lars_apply_kernel(CollDev d, size_t poff, size_t nvec, const float* __restrict__ scratch,
                                                                  const int4* __restrict__ seg, int nseg, const float2* __restrict__ scal,
                                                                  const float* __restrict__ hp, float* __restrict__ master,
                                                                  float* __restrict__ mom, int chan) {
  float* const state[2] = {master, mom};
  fused_step<DT, MODE>(d, LarsGrad{scratch, seg, nseg, scal}, poff, nvec, LarsOpt<DT == BNET_BF16 ? 1 : 2>{hp[optim::kLarsLr], hp[optim::kLarsMomentum]},
                       state, 0, chan);
}

// ------------------------------------------------------------------ exponential moving average of the master weights
// One batch of the EMA update: U float4s of the master shard (and of the EMA shard unless COPY) per thread, every load
// issued before any math, non-temporal as in fused_batch.
template <int U, bool COPY>
__device__ __forceinline__ void ema_batch(const float4* __restrict__ master, float4* __restrict__ ema, size_t i, size_t stride,
                                          float w) {
  float4 m[U], e[COPY ? 1 : U];
#pragma unroll
  for (int u = 0; u < U; u++) m[u] = ptx::ld_na_f4(master + i + u * stride);
  if constexpr (!COPY) {
#pragma unroll
    for (int u = 0; u < U; u++) e[u] = ptx::ld_na_f4(ema + i + u * stride);
  }
#pragma unroll
  for (int u = 0; u < U; u++) {
    float4 r = m[u];
    if constexpr (!COPY) {
      r.x = optim::ema_lerp(e[u].x, m[u].x, w); r.y = optim::ema_lerp(e[u].y, m[u].y, w);
      r.z = optim::ema_lerp(e[u].z, m[u].z, w); r.w = optim::ema_lerp(e[u].w, m[u].w, w);
    }
    ptx::st_na_f4(ema + i + u * stride, r);
  }
}

template <bool COPY>
__device__ __forceinline__ void ema_body(const float4* __restrict__ master, float4* __restrict__ ema, size_t n4, float w) {
  constexpr int U = 4;
  const size_t stride = (size_t)gridDim.x * kThreads;
  size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
  for (; i + (U - 1) * stride < n4; i += U * stride) ema_batch<U, COPY>(master, ema, i, stride, w);
  for (; i < n4; i += stride) ema_batch<1, COPY>(master, ema, i, stride, w);
}

// Per bucket, after the optimizer step's last update launch: on an EMA step (optim::ema_gate on the block), this rank's
// fp32 EMA shard becomes a copy of the master shard (no update averaged yet) or lerp(ema, master, weight).  On any other
// step every thread exits after reading the block, before touching either shard.  Rank-local, no barriers, no atomics:
// each element's bits depend on neither the grid nor a repeat.
__global__ void __launch_bounds__(kThreads) bnet_ema_update_kernel(const float4* __restrict__ master, float4* __restrict__ ema,
                                                                  size_t n4, const float* __restrict__ blk) {
  const optim::EmaGate g = optim::ema_gate(blk[optim::kEmaStep], blk[optim::kEmaEvery], blk[optim::kEmaNAveraged]);
  if (!g.update) return;
  if (g.copy) ema_body<true>(master, ema, n4, 0.0f);
  else ema_body<false>(master, ema, n4, blk[optim::kEmaWeight]);
}

// Once per optimizer step, one thread, after every bucket's bnet_ema_update_kernel: count the step, and the update when
// it was an EMA step.  A kernel, not a host-side add, because the second increment depends on device values.
__global__ void bnet_ema_advance_kernel(float* __restrict__ blk) {
  const optim::EmaGate g = optim::ema_gate(blk[optim::kEmaStep], blk[optim::kEmaEvery], blk[optim::kEmaNAveraged]);
  if (g.update) blk[optim::kEmaNAveraged] += 1.0f;
  blk[optim::kEmaStep] += 1.0f;
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
    // max and min never use the switch, whatever `algo` asks: the peer-load, one-shot and LL kernels all combine with
    // fmaxf / fminf (a NaN loses to a number), and multimem's min / max has no f32 form and no
    // documented NaN rule, so a result's NaNs would depend on the dtype, the world size and the message size.
    case BNET_MAX: return launch(bnet_allreduce_p2p_kernel<DT, BNET_MAX>, nb, kThreads, st, c->devp, off, nvec, chan);
    case BNET_MIN: return launch(bnet_allreduce_p2p_kernel<DT, BNET_MIN>, nb, kThreads, st, c->devp, off, nvec, chan);
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
  if (offset + bytes > c->alloc_bytes - kPadBytes) return fail("one-shot all-reduce range outside the heap");
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

// Each optimizer's fused kernel, by dtype and MODE
struct SgdKernel {
  template <int DT, int MODE> static constexpr auto fn = bnet_fused_sgd_kernel<DT, MODE>;
};
struct AdamWKernel {
  template <int DT, int MODE> static constexpr auto fn = bnet_fused_adamw_kernel<DT, MODE>;
};

// What a fused optimizer launch needs once its input has been checked
struct FusedLaunch {
  size_t goff, poff, nvec;   // heap byte offsets of gradients and parameters, 16-byte vectors in the bucket
  bool nvls;                 // in-switch reduction (MODE 1) when there is more than one rank
  int nb;
  cudaStream_t st;
};

// Input checks and launch set-up of the fused optimizer entry points: `what` names the optimizer in the messages,
// `state` lists its fp32 arrays.
static int fused_prologue(BnetColl* c, const char* what, size_t grad_off, size_t param_off, size_t count, int dtype,
                          int channel, std::initializer_list<const float*> state, int nblocks, void* stream, FusedLaunch& f) {
  if (channel < 0 || channel >= BNET_COLL_CHANNELS) return fail("bad channel");
  if (dtype != BNET_F32 && dtype != BNET_BF16) return fail("fused %s supports f32 and bf16", what);
  size_t bytes = count * elsize(dtype);
  if (bytes % (16 * (size_t)c->world) || grad_off % 16 || param_off % 16) return fail("fused %s needs 16-byte aligned offsets and bytes%%(16*world)==0", what);
  if (grad_off + bytes > c->alloc_bytes - kPadBytes || param_off + bytes > c->alloc_bytes - kPadBytes) return fail("fused %s range outside the heap", what);
  uintptr_t addr = 0;
  for (const float* s : state) addr |= (uintptr_t)s;
  if (addr & 15) return fail("optimizer state must be 16-byte aligned");
  refresh_devp(c);
  f.goff = kPadBytes + grad_off;
  f.poff = kPadBytes + param_off;
  f.nvec = bytes / 16;
  f.nvls = prefer_nvls(c) && env_int("FUSED_NVLS", 1);
  f.nb = pick_blocks(c, f.nvec / c->world, nblocks, f.nvls ? BLK_FUSED_NVLS : BLK_P2P);
  f.st = (cudaStream_t)stream;
  return 0;
}

// Launches K's kernel for `dtype` in MODE 0 on one GPU, 1 with NVLS, 2 with peer loads and stores, with `args` after
// the communicator.
template <class K, typename... A>
static int run_fused_kernel(BnetColl* c, int dtype, const FusedLaunch& f, A... args) {
  const int mode = c->world == 1 ? 0 : f.nvls ? 1 : 2;
  const std::decay_t<decltype(K::template fn<BNET_F32, 0>)> kern[2][3] = {
      {K::template fn<BNET_F32, 0>, K::template fn<BNET_F32, 1>, K::template fn<BNET_F32, 2>},
      {K::template fn<BNET_BF16, 0>, K::template fn<BNET_BF16, 1>, K::template fn<BNET_BF16, 2>}};
  return launch(kern[dtype == BNET_BF16][mode], f.nb, kThreads, f.st, c->devp, args...);
}
// The one-kernel steps: gradient and parameter offsets and the vector count first.
template <class K, typename... A>
static int run_fused(BnetColl* c, int dtype, const FusedLaunch& f, A... args) {
  return run_fused_kernel<K>(c, dtype, f, f.goff, f.poff, f.nvec, args...);
}

BNET_API int bnet_fused_allreduce_sgd(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype, float lr,
                                      float momentum, float weight_decay, float grad_scale, float* master,
                                      float* mom_buf, int zero_grads, int channel, int nblocks, void* stream) {
  FusedLaunch f;
  if (fused_prologue(c, "SGD", grad_off, param_off, count, dtype, channel, {master, mom_buf}, nblocks, stream, f) < 0) return -1;
  return run_fused<SgdKernel>(c, dtype, f, lr, momentum, weight_decay, grad_scale, master, mom_buf, zero_grads, channel,
                              (const float*)nullptr);
}

// Same, with {lr, momentum, weight_decay, grad_scale} read from 4 floats of device memory at kernel run time.
BNET_API int bnet_fused_allreduce_sgd_hp(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype,
                                         const float* hp_dev, float* master, float* mom_buf, int zero_grads, int channel,
                                         int nblocks, void* stream) {
  if (!hp_dev || ((uintptr_t)hp_dev & 15)) return fail("hyper-parameter block must be a 16-byte aligned device pointer");
  FusedLaunch f;
  if (fused_prologue(c, "SGD", grad_off, param_off, count, dtype, channel, {master, mom_buf}, nblocks, stream, f) < 0) return -1;
  return run_fused<SgdKernel>(c, dtype, f, 0.f, 0.f, 0.f, 1.f, master, mom_buf, zero_grads, channel, hp_dev);
}

BNET_API int bnet_fused_allreduce_adamw(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype,
                                        const float* hp_dev, float* master, float* exp_avg, float* exp_avg_sq, int zero_grads,
                                        int channel, int nblocks, void* stream) {
  if (!hp_dev || ((uintptr_t)hp_dev & 15)) return fail("hyper-parameter block must be a 16-byte aligned device pointer");
  FusedLaunch f;
  if (fused_prologue(c, "AdamW", grad_off, param_off, count, dtype, channel, {master, exp_avg, exp_avg_sq}, nblocks, stream, f) < 0)
    return -1;
  return run_fused<AdamWKernel>(c, dtype, f, hp_dev, master, exp_avg, exp_avg_sq, zero_grads, channel);
}

// ---- gradient clipping by global norm: the three stages of the clipped step
struct ClipNormKernel {
  template <int DT, int MODE> static constexpr auto fn = bnet_clip_norm_kernel<DT, MODE>;
};
struct AccumNormKernel {
  template <int DT, int MODE> static constexpr auto fn = bnet_accum_norm_kernel<DT, MODE>;
};
struct ClipSgdKernel {
  template <int DT, int MODE> static constexpr auto fn = bnet_clip_apply_sgd_kernel<DT, MODE>;
};
struct ClipAdamWKernel {
  template <int DT, int MODE> static constexpr auto fn = bnet_clip_apply_adamw_kernel<DT, MODE>;
};

static int clip_block_check(const float* clip) {
  if (!clip || ((uintptr_t)clip & 15)) return fail("clip block must be a 16-byte aligned device pointer");
  return 0;
}

BNET_API int bnet_fused_clip_reduce_norm(BnetColl* c, size_t grad_off, size_t count, int dtype, float* scratch, double* partial,
                                         int channel, int nblocks, void* stream) {
  if (!partial || ((uintptr_t)partial & 7)) return fail("partial row must be an 8-byte aligned device pointer");
  FusedLaunch f;
  if (fused_prologue(c, "clip norm", grad_off, grad_off, count, dtype, channel, {scratch}, nblocks, stream, f) < 0) return -1;
  return run_fused_kernel<ClipNormKernel>(c, dtype, f, f.goff, f.nvec, scratch, partial, channel);
}

BNET_API int bnet_fused_accum_reduce_norm(BnetColl* c, size_t grad_off, size_t count, int dtype, float* scratch, double* partial,
                                          int channel, int nblocks, void* stream) {
  if (!partial || ((uintptr_t)partial & 7)) return fail("partial row must be an 8-byte aligned device pointer");
  FusedLaunch f;
  if (fused_prologue(c, "accumulating norm", grad_off, grad_off, count, dtype, channel, {scratch}, nblocks, stream, f) < 0) return -1;
  return run_fused_kernel<AccumNormKernel>(c, dtype, f, f.goff, f.nvec, scratch, partial, channel);
}

BNET_API int bnet_fused_clip_coef(BnetColl* c, const double* partials, int nrows, size_t xchg_off, float grad_scale, float* clip,
                                  int channel, void* stream) {
  if (channel < 0 || channel >= BNET_COLL_CHANNELS) return fail("bad channel");
  if (nrows < 1 || !partials || ((uintptr_t)partials & 7)) return fail("clip coefficient needs >= 1 partial row, 8-byte aligned");
  if (clip_block_check(clip) < 0) return -1;
  if (xchg_off % 16 || xchg_off + (size_t)c->world * sizeof(double) > c->alloc_bytes - kPadBytes)
    return fail("clip exchange area must be 16-byte aligned and inside the heap");
  refresh_devp(c);
  return launch(bnet_clip_coef_kernel, 1, kThreads, (cudaStream_t)stream, c->devp, partials,
                (size_t)nrows * BNET_COLL_MAX_BLOCKS, kPadBytes + xchg_off, grad_scale, clip, channel);
}

BNET_API int bnet_fused_clip_apply_sgd(BnetColl* c, size_t param_off, size_t count, int dtype, const float* scratch,
                                       const float* clip, float lr, float momentum, float weight_decay, float grad_scale,
                                       float* master, float* mom_buf, int channel, int nblocks, void* stream) {
  if (clip_block_check(clip) < 0) return -1;
  FusedLaunch f;
  if (fused_prologue(c, "clipped SGD", param_off, param_off, count, dtype, channel, {scratch, master, mom_buf}, nblocks, stream, f) < 0)
    return -1;
  return run_fused_kernel<ClipSgdKernel>(c, dtype, f, f.poff, f.nvec, scratch, clip, lr, momentum, weight_decay, grad_scale, master,
                                         mom_buf, channel, (const float*)nullptr);
}

BNET_API int bnet_fused_clip_apply_sgd_hp(BnetColl* c, size_t param_off, size_t count, int dtype, const float* scratch,
                                          const float* clip, const float* hp_dev, float* master, float* mom_buf, int channel,
                                          int nblocks, void* stream) {
  if (!hp_dev || ((uintptr_t)hp_dev & 15)) return fail("hyper-parameter block must be a 16-byte aligned device pointer");
  if (clip_block_check(clip) < 0) return -1;
  FusedLaunch f;
  if (fused_prologue(c, "clipped SGD", param_off, param_off, count, dtype, channel, {scratch, master, mom_buf}, nblocks, stream, f) < 0)
    return -1;
  return run_fused_kernel<ClipSgdKernel>(c, dtype, f, f.poff, f.nvec, scratch, clip, 0.f, 0.f, 0.f, 1.f, master, mom_buf, channel,
                                         hp_dev);
}

BNET_API int bnet_fused_clip_apply_adamw(BnetColl* c, size_t param_off, size_t count, int dtype, const float* scratch,
                                         const float* clip, const float* hp_dev, float* master, float* exp_avg, float* exp_avg_sq,
                                         int channel, int nblocks, void* stream) {
  if (!hp_dev || ((uintptr_t)hp_dev & 15)) return fail("hyper-parameter block must be a 16-byte aligned device pointer");
  if (clip_block_check(clip) < 0) return -1;
  FusedLaunch f;
  if (fused_prologue(c, "clipped AdamW", param_off, param_off, count, dtype, channel, {scratch, master, exp_avg, exp_avg_sq}, nblocks,
                     stream, f) < 0)
    return -1;
  return run_fused_kernel<ClipAdamWKernel>(c, dtype, f, f.poff, f.nvec, scratch, clip, hp_dev, master, exp_avg, exp_avg_sq, channel);
}

// ---- parameter groups: the SGD and AdamW steps with per-group lr and weight decay (tables validated by the caller)
struct SgdGroupsKernel {
  template <int DT, int MODE> static constexpr auto fn = bnet_fused_sgd_groups_kernel<DT, MODE>;
};
struct AdamWGroupsKernel {
  template <int DT, int MODE> static constexpr auto fn = bnet_fused_adamw_groups_kernel<DT, MODE>;
};
struct ClipSgdGroupsKernel {
  template <int DT, int MODE> static constexpr auto fn = bnet_clip_apply_sgd_groups_kernel<DT, MODE>;
};
struct ClipAdamWGroupsKernel {
  template <int DT, int MODE> static constexpr auto fn = bnet_clip_apply_adamw_groups_kernel<DT, MODE>;
};
static_assert(sizeof(BnetGroupSeg) == sizeof(int4), "group segment rows are int4");

static int groups_check(const float* hp_dev, const float* groups, int ngroups, const BnetGroupSeg* segs, int nseg) {
  if (!hp_dev || ((uintptr_t)hp_dev & 15)) return fail("hyper-parameter block must be a 16-byte aligned device pointer");
  if (ngroups < 1 || ngroups > BNET_GROUPS_MAX || !groups || ((uintptr_t)groups & 15))
    return fail("group table needs 1..%d rows, 16-byte aligned (got %d)", BNET_GROUPS_MAX, ngroups);
  if (nseg < 1 || !segs || ((uintptr_t)segs & 15)) return fail("group segment table needs >= 1 row, 16-byte aligned");
  return 0;
}

BNET_API int bnet_fused_allreduce_sgd_groups(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype,
                                             const float* hp_dev, const float* groups, int ngroups, const BnetGroupSeg* segs,
                                             int nseg, float* master, float* mom_buf, int zero_grads, int channel, int nblocks,
                                             void* stream) {
  if (groups_check(hp_dev, groups, ngroups, segs, nseg) < 0) return -1;
  FusedLaunch f;
  if (fused_prologue(c, "grouped SGD", grad_off, param_off, count, dtype, channel, {master, mom_buf}, nblocks, stream, f) < 0) return -1;
  return run_fused<SgdGroupsKernel>(c, dtype, f, hp_dev, reinterpret_cast<const float4*>(groups), ngroups,
                                    reinterpret_cast<const int4*>(segs), nseg, master, mom_buf, zero_grads, channel);
}

BNET_API int bnet_fused_allreduce_adamw_groups(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype,
                                               const float* hp_dev, const float* groups, int ngroups, const BnetGroupSeg* segs,
                                               int nseg, float* master, float* exp_avg, float* exp_avg_sq, int zero_grads,
                                               int channel, int nblocks, void* stream) {
  if (groups_check(hp_dev, groups, ngroups, segs, nseg) < 0) return -1;
  FusedLaunch f;
  if (fused_prologue(c, "grouped AdamW", grad_off, param_off, count, dtype, channel, {master, exp_avg, exp_avg_sq}, nblocks, stream,
                     f) < 0)
    return -1;
  return run_fused<AdamWGroupsKernel>(c, dtype, f, hp_dev, reinterpret_cast<const float4*>(groups), ngroups,
                                      reinterpret_cast<const int4*>(segs), nseg, master, exp_avg, exp_avg_sq, zero_grads, channel);
}

BNET_API int bnet_fused_clip_apply_sgd_groups(BnetColl* c, size_t param_off, size_t count, int dtype, const float* scratch,
                                              const float* clip, const float* hp_dev, const float* groups, int ngroups,
                                              const BnetGroupSeg* segs, int nseg, float* master, float* mom_buf, int channel,
                                              int nblocks, void* stream) {
  if (groups_check(hp_dev, groups, ngroups, segs, nseg) < 0 || clip_block_check(clip) < 0) return -1;
  FusedLaunch f;
  if (fused_prologue(c, "clipped grouped SGD", param_off, param_off, count, dtype, channel, {scratch, master, mom_buf}, nblocks,
                     stream, f) < 0)
    return -1;
  return run_fused_kernel<ClipSgdGroupsKernel>(c, dtype, f, f.poff, f.nvec, scratch, clip, hp_dev, reinterpret_cast<const float4*>(groups),
                                               ngroups, reinterpret_cast<const int4*>(segs), nseg, master, mom_buf, channel);
}

BNET_API int bnet_fused_clip_apply_adamw_groups(BnetColl* c, size_t param_off, size_t count, int dtype, const float* scratch,
                                                const float* clip, const float* hp_dev, const float* groups, int ngroups,
                                                const BnetGroupSeg* segs, int nseg, float* master, float* exp_avg,
                                                float* exp_avg_sq, int channel, int nblocks, void* stream) {
  if (groups_check(hp_dev, groups, ngroups, segs, nseg) < 0 || clip_block_check(clip) < 0) return -1;
  FusedLaunch f;
  if (fused_prologue(c, "clipped grouped AdamW", param_off, param_off, count, dtype, channel, {scratch, master, exp_avg, exp_avg_sq},
                     nblocks, stream, f) < 0)
    return -1;
  return run_fused_kernel<ClipAdamWGroupsKernel>(c, dtype, f, f.poff, f.nvec, scratch, clip, hp_dev,
                                                 reinterpret_cast<const float4*>(groups), ngroups, reinterpret_cast<const int4*>(segs),
                                                 nseg, master, exp_avg, exp_avg_sq, channel);
}

// ---- LARS: norm, trust and apply stages (the tables themselves are validated by the caller before upload)
struct LarsApplyKernel {
  template <int DT, int MODE> static constexpr auto fn = bnet_lars_apply_kernel<DT, MODE>;
};
static_assert(sizeof(BnetLarsSeg) == sizeof(int4) && sizeof(BnetLarsTensor) == sizeof(int4), "LARS tables are int4 rows");

static int lars_seg_check(const BnetLarsSeg* segs, int nseg) {
  if (nseg < 1 || !segs || ((uintptr_t)segs & 15)) return fail("LARS segment table needs >= 1 row, 16-byte aligned");
  return 0;
}

BNET_API int bnet_fused_lars_norm(BnetColl* c, size_t count, int dtype, const float* master, const float* scratch,
                                  const BnetLarsSeg* segs, int nseg, double* slots, int nslots, int nblocks, void* stream) {
  if (dtype != BNET_F32 && dtype != BNET_BF16) return fail("LARS norm supports f32 and bf16");
  if ((count * elsize(dtype)) % (16 * (size_t)c->world)) return fail("LARS norm needs bytes%%(16*world)==0");
  if (((uintptr_t)master | (uintptr_t)scratch | (uintptr_t)slots) & 15) return fail("LARS norm buffers must be 16-byte aligned");
  if (lars_seg_check(segs, nseg) < 0) return -1;
  if (nslots < 1) return fail("LARS norm needs >= 1 slot");
  int nb = nblocks > 0 ? nblocks : (int)env_int("COLL_BLOCKS_SINGLE", 264);
  if (nb > nslots) nb = nslots;
  if (nb > BNET_COLL_MAX_BLOCKS) nb = BNET_COLL_MAX_BLOCKS;
  return launch(bnet_lars_norm_kernel, nb, kThreads, (cudaStream_t)stream, reinterpret_cast<const float4*>(master),
                reinterpret_cast<const float4*>(scratch), reinterpret_cast<const int4*>(segs), nseg, dtype == BNET_BF16 ? 2 : 1,
                reinterpret_cast<double2*>(slots), nslots);
}

BNET_API int bnet_fused_lars_trust(BnetColl* c, const double* slots, const BnetLarsTensor* tensors, int ntensors, size_t xchg_off,
                                   const float* clip, const float* hp, float* scal, float* trust, int channel, void* stream) {
  if (channel < 0 || channel >= BNET_COLL_CHANNELS) return fail("bad channel");
  if (ntensors < 1 || !tensors || ((uintptr_t)tensors & 15)) return fail("LARS tensor table needs >= 1 row, 16-byte aligned");
  if (!slots || ((uintptr_t)slots & 15)) return fail("LARS slots must be a 16-byte aligned device pointer");
  if (clip_block_check(clip) < 0) return -1;
  if (!hp || ((uintptr_t)hp & 15)) return fail("hyper-parameter block must be a 16-byte aligned device pointer");
  if (!scal || ((uintptr_t)scal & 7) || !trust || ((uintptr_t)trust & 3)) return fail("LARS outputs must be aligned device pointers");
  if (xchg_off % 16 || xchg_off + 2 * (size_t)c->world * ntensors * sizeof(double) > c->alloc_bytes - kPadBytes)
    return fail("LARS exchange area must be 16-byte aligned and inside the heap");
  refresh_devp(c);
  return launch(bnet_lars_trust_kernel, 1, kThreads, (cudaStream_t)stream, c->devp, reinterpret_cast<const double2*>(slots),
                reinterpret_cast<const int4*>(tensors), ntensors, kPadBytes + xchg_off, clip, hp, reinterpret_cast<float2*>(scal),
                trust, channel);
}

BNET_API int bnet_fused_lars_apply(BnetColl* c, size_t param_off, size_t count, int dtype, const float* scratch, const BnetLarsSeg* segs,
                                   int nseg, const float* scal, const float* hp, float* master, float* mom_buf, int channel, int nblocks,
                                   void* stream) {
  if (!hp || ((uintptr_t)hp & 15)) return fail("hyper-parameter block must be a 16-byte aligned device pointer");
  if (lars_seg_check(segs, nseg) < 0) return -1;
  if (!scal || ((uintptr_t)scal & 7)) return fail("LARS scalars must be an 8-byte aligned device pointer");
  FusedLaunch f;
  if (fused_prologue(c, "LARS", param_off, param_off, count, dtype, channel, {scratch, master, mom_buf}, nblocks, stream, f) < 0)
    return -1;
  return run_fused_kernel<LarsApplyKernel>(c, dtype, f, f.poff, f.nvec, scratch, reinterpret_cast<const int4*>(segs), nseg,
                                           reinterpret_cast<const float2*>(scal), hp, master, mom_buf, channel);
}

// ---- exponential moving average of the master weights
static int ema_block_check(const float* blk) {
  if (!blk || ((uintptr_t)blk & 15)) return fail("EMA block must be a 16-byte aligned device pointer");
  return 0;
}

BNET_API int bnet_ema_update(BnetColl* c, size_t count, const float* master, float* ema, const float* blk, int nblocks, void* stream) {
  if (count == 0 || count % 4) return fail("EMA update needs a whole number (>= 1) of float4s");
  if (((uintptr_t)master | (uintptr_t)ema) & 15) return fail("EMA shards must be 16-byte aligned");
  if (ema_block_check(blk) < 0) return -1;
  const size_t n4 = count / 4;
  int nb = nblocks;
  if (nb <= 0) {   // two CTAs per SM, no more than give every thread one batch of 4 vectors
    nb = (int)env_int("COLL_BLOCKS_SINGLE", 264);
    const size_t want = (n4 + kThreads * 4 - 1) / (kThreads * 4);
    if ((size_t)nb > want) nb = (int)want;
  }
  if (nb > BNET_COLL_MAX_BLOCKS) nb = BNET_COLL_MAX_BLOCKS;
  if (nb < 1) nb = 1;
  return launch(bnet_ema_update_kernel, nb, kThreads, (cudaStream_t)stream, reinterpret_cast<const float4*>(master),
                reinterpret_cast<float4*>(ema), n4, blk);
}

BNET_API int bnet_ema_advance(BnetColl* c, float* blk, void* stream) {
  if (ema_block_check(blk) < 0) return -1;
  return launch(bnet_ema_advance_kernel, 1, 1, (cudaStream_t)stream, blk);
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

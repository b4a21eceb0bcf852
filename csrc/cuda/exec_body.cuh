// The data-movement bodies of the transport executor (csrc/cuda/nvl_exec.cu): what ONE CTA does with its share
// of a job — copy (K1), move + accumulate (K4), move + cast (K5), fp8 gradient compression.
//
// Written as functions of (tid, nthreads) with the PTX accesses behind __CUDA_ARCH__ switches, so that the
// SAME code is inlined into the sm_90a kernels by nvcc and compiled by g++ for csrc/tests/exec_emu_test.cc,
// which walks an emulated CTA over every op, size and alignment on the CPU (`make test`, no GPU needed).
//
// Memory-level parallelism: every vector loop is `batched<U>` — U 16-byte loads are issued before the first
// dependent instruction (the reductions/stores that follow are fire-and-forget).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "cuda/exec_ops.h"

#if defined(__CUDACC__)
#define BNET_XD __host__ __device__ __forceinline__
#define BNET_XD_FN __host__ __device__ inline
#else
#define BNET_XD inline
#define BNET_XD_FN inline
#endif

namespace bnet {
namespace cuda {

BNET_XD bool op_is_e5m2(uint32_t op) { return (op >= OP_CAST_BF16_TO_E5M2 && op <= OP_CAST_F32_TO_E5M2) || op == OP_CAST_E5M2_TO_F32; }

namespace xb {   // access primitives: PTX on the device, plain C++ in the emulation

BNET_XD int4 ld16(const int4* p) {
#if defined(__CUDA_ARCH__)
  int4 r;
  asm volatile("ld.global.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
#else
  int4 r;
  memcpy(&r, p, 16);
  return r;
#endif
}
BNET_XD void st16(int4* p, const int4& v) {
#if defined(__CUDA_ARCH__)
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
#else
  memcpy(p, &v, 16);
#endif
}
BNET_XD float4 ld16f(const float4* p) {
#if defined(__CUDA_ARCH__)
  float4 r;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
  return r;
#else
  float4 r;
  memcpy(&r, p, 16);
  return r;
#endif
}
BNET_XD void st16f(float4* p, const float4& v) {
#if defined(__CUDA_ARCH__)
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
#else
  memcpy(p, &v, 16);
#endif
}
BNET_XD uint2 ld8(const void* p) {          // p is 8-byte aligned
#if defined(__CUDA_ARCH__)
  return *reinterpret_cast<const uint2*>(p);
#else
  uint2 r;
  memcpy(&r, p, 8);
  return r;
#endif
}
BNET_XD uint32_t ld4(const void* p) {       // p is 4-byte aligned
#if defined(__CUDA_ARCH__)
  return *reinterpret_cast<const uint32_t*>(p);
#else
  uint32_t r;
  memcpy(&r, p, 4);
  return r;
#endif
}
BNET_XD void st8(void* p, const uint2& v) {  // p is 8-byte aligned
#if defined(__CUDA_ARCH__)
  *reinterpret_cast<uint2*>(p) = v;
#else
  memcpy(p, &v, 8);
#endif
}
// fire-and-forget reductions at system scope (one packet over NVLink, no return value).  The host versions are atomic too
// (compare-and-swap on the element's bits): in the emulation several sender PROCESSES may accumulate into one shared
// buffer at the same time, exactly like several GPUs into one output (csrc/coll/transport_mesh.cc).
#if !defined(__CUDA_ARCH__)
inline void host_atomic_add_f32(float* p, float v) {
  uint32_t* u = reinterpret_cast<uint32_t*>(p);
  uint32_t old = __atomic_load_n(u, __ATOMIC_RELAXED), want;
  do {
    float f;
    memcpy(&f, &old, 4);
    f += v;
    memcpy(&want, &f, 4);
  } while (!__atomic_compare_exchange_n(u, &old, want, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED));
}
inline void host_atomic_add_bf16(__nv_bfloat16* p, __nv_bfloat16 v) {
  uint16_t* u = reinterpret_cast<uint16_t*>(p);
  uint16_t old = __atomic_load_n(u, __ATOMIC_RELAXED), want;
  do {
    __nv_bfloat16 b;
    memcpy((void*)&b, &old, 2);
    b = __float2bfloat16(__bfloat162float(b) + __bfloat162float(v));
    memcpy(&want, (const void*)&b, 2);
  } while (!__atomic_compare_exchange_n(u, &old, want, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED));
}
#endif
BNET_XD void red_f32(float* p, float v) {
#if defined(__CUDA_ARCH__)
  asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
#else
  host_atomic_add_f32(p, v);
#endif
}
BNET_XD void red_v4_f32(float* p, const float4& v) {
#if defined(__CUDA_ARCH__)
  asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
#else
  host_atomic_add_f32(p, v.x); host_atomic_add_f32(p + 1, v.y); host_atomic_add_f32(p + 2, v.z); host_atomic_add_f32(p + 3, v.w);
#endif
}
BNET_XD void red_bf16(__nv_bfloat16* p, __nv_bfloat16 v) {
#if defined(__CUDA_ARCH__)
  atomicAdd(p, v);
#else
  host_atomic_add_bf16(p, v);
#endif
}
BNET_XD void red_v4_bf16x2(uint32_t* p, const int4& v) {
#if defined(__CUDA_ARCH__)
  asm volatile("red.relaxed.sys.global.add.noftz.v4.bf16x2 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
#else
  __nv_bfloat16 s[8];
  memcpy((void*)s, &v, 16);
  __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(p);
  for (int k = 0; k < 8; k++) red_bf16(d + k, s[k]);
#endif
}

// U independent 16/32-byte loads in flight per thread, then the dependent work
template <int U, typename Raw, typename Load, typename Use>
BNET_XD void batched(size_t nvec, int tid, int nthreads, Load load, Use use) {
  size_t i = (size_t)tid;
  const size_t stride = (size_t)nthreads;
  for (; i + (U - 1) * stride < nvec; i += U * stride) {
    Raw v[U];
#pragma unroll
    for (int u = 0; u < U; u++) v[u] = load(i + u * stride);
#pragma unroll
    for (int u = 0; u < U; u++) use(i + u * stride, v[u]);
  }
  for (; i < nvec; i += stride) use(i, load(i));
}

struct F8 { float4 lo, hi; };   // 8 floats = two 16-byte loads

BNET_XD void unpack_bf16x8(const int4& v, float4* lo, float4* hi) {
  __nv_bfloat162 h[4];
  memcpy((void*)h, &v, 16);
  float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]);
  float2 c = __bfloat1622float2(h[2]), e = __bfloat1622float2(h[3]);
  *lo = make_float4(a.x, a.y, b.x, b.y);
  *hi = make_float4(c.x, c.y, e.x, e.y);
}

}  // namespace xb

// source bytes per indivisible work unit (keeps CTA / chunk cuts vector-aligned on BOTH sides)
BNET_XD size_t src_unit_for(uint32_t op) {
  if (op == OP_CAST_F32_TO_BF16 || op == OP_CAST_BF16_TO_E4M3 || op == OP_CAST_BF16_TO_E5M2 || op == OP_RED_ADD_F32) return 32;
  if (op == OP_CAST_F32_TO_E4M3 || op == OP_CAST_F32_TO_E5M2) return 64;
  return 16;
}

// destination offset that corresponds to a source offset
BNET_XD size_t dst_offset_for(uint32_t op, size_t src_off) {
  if (op == OP_CAST_BF16_TO_F32 || op == OP_ACC_BF16_TO_F32) return src_off * 2;
  if (op == OP_CAST_F32_TO_BF16 || op == OP_CAST_BF16_TO_E4M3 || op == OP_CAST_BF16_TO_E5M2) return src_off / 2;
  if (op == OP_ACC_E4M3_TO_F32 || op == OP_ACC_E5M2_TO_F32 || op == OP_CAST_E4M3_TO_F32 || op == OP_CAST_E5M2_TO_F32) return src_off * 4;
  if (op == OP_CAST_F32_TO_E4M3 || op == OP_CAST_F32_TO_E5M2) return src_off / 4;
  return src_off;
}

// Every CTA of a cluster takes a contiguous share [b0, b1) of the job's source bytes, cut at multiples of the
// op's work unit so that both the source and the destination side of every share stay vector aligned.
BNET_XD void cta_share(uint32_t op, size_t nbytes, uint32_t crank, uint32_t csize, size_t* b0, size_t* b1) {
  const size_t unit = src_unit_for(op);
  const size_t units = (nbytes + unit - 1) / unit;
  const size_t per = (units + csize - 1) / csize;
  size_t lo = (size_t)crank * per * unit, hi = lo + per * unit;
  if (lo > nbytes) lo = nbytes;
  if (hi > nbytes) hi = nbytes;
  *b0 = lo;
  *b1 = hi;
}

// Moves/reduces [0,n) source bytes for one CTA's share.  tid/nthreads are CTA-local.
BNET_XD_FN void process_range(uint32_t op, const char* src, char* dst, size_t n, int tid, int nthreads, float scale = 1.0f) {
  if (n == 0) return;
  if (op == OP_COPY) {
    // align the destination, then go wide if the source agrees
    size_t head = (16 - ((uintptr_t)dst & 15)) & 15;
    if (head > n) head = n;
    for (size_t i = tid; i < head; i += nthreads) dst[i] = src[i];
    src += head; dst += head; n -= head;
    if (((uintptr_t)src & 15) == 0) {
      const size_t nvec = n >> 4;
      const int4* s = reinterpret_cast<const int4*>(src);
      int4* d = reinterpret_cast<int4*>(dst);
      xb::batched<8, int4>(nvec, tid, nthreads, [&](size_t i) { return xb::ld16(s + i); },
                           [&](size_t i, const int4& v) { xb::st16(d + i, v); });
      for (size_t i = (nvec << 4) + tid; i < n; i += nthreads) dst[i] = src[i];
    } else if ((((uintptr_t)src ^ (uintptr_t)dst) & 3) == 0) {
      size_t n4 = n >> 2;
      const uint32_t* s4 = (const uint32_t*)src;
      uint32_t* d4 = (uint32_t*)dst;
      for (size_t i = tid; i < n4; i += nthreads) d4[i] = s4[i];
      for (size_t i = (n4 << 2) + tid; i < n; i += nthreads) dst[i] = src[i];
    } else {
      for (size_t i = tid; i < n; i += nthreads) dst[i] = src[i];
    }
    return;
  }
  if (op == OP_RED_ADD_F32) {
    size_t ne = n >> 2;
    const float* s = (const float*)src;
    float* d = (float*)dst;
    if ((((uintptr_t)s | (uintptr_t)d) & 15) == 0) {
      size_t nv = ne >> 2;
      xb::batched<8, float4>(nv, tid, nthreads, [&](size_t i) { return xb::ld16f(reinterpret_cast<const float4*>(s) + i); },
                             [&](size_t i, const float4& v) { xb::red_v4_f32(d + 4 * i, v); });   // 16-byte reduction packets
      for (size_t i = (nv << 2) + tid; i < ne; i += nthreads) xb::red_f32(d + i, s[i]);
    } else {
      for (size_t i = tid; i < ne; i += nthreads) xb::red_f32(d + i, s[i]);
    }
    return;
  }
  if (op == OP_RED_ADD_BF16) {
    size_t ne = n >> 1;
    const __nv_bfloat16* s = (const __nv_bfloat16*)src;
    __nv_bfloat16* d = (__nv_bfloat16*)dst;
    if ((((uintptr_t)s | (uintptr_t)d) & 15) == 0) {
      size_t nv = ne >> 3;
      xb::batched<8, int4>(nv, tid, nthreads, [&](size_t i) { return xb::ld16(reinterpret_cast<const int4*>(s) + i); },
                           [&](size_t i, const int4& v) { xb::red_v4_bf16x2(reinterpret_cast<uint32_t*>(d) + 4 * i, v); });
      for (size_t i = (nv << 3) + tid; i < ne; i += nthreads) xb::red_bf16(d + i, s[i]);
    } else {
      for (size_t i = tid; i < ne; i += nthreads) xb::red_bf16(d + i, s[i]);
    }
    return;
  }
  if (op == OP_CAST_BF16_TO_F32 || op == OP_ACC_BF16_TO_F32) {
    size_t ne = n >> 1;
    const __nv_bfloat16* s = (const __nv_bfloat16*)src;
    float* d = (float*)dst;
    const bool acc = op == OP_ACC_BF16_TO_F32;
    if ((((uintptr_t)s | (uintptr_t)d) & 15) == 0) {
      size_t nv = ne >> 3;   // 8 bf16 in, 2 x float4 out
      // Lane-interleaved inside blocks of 32 vectors (256 elements): vector l of a block takes elements [4l, 4l+4) and
      // [128+4l, 128+4l+4).  Each of a warp's two output instructions then covers 512 CONTIGUOUS bytes (whole sectors,
      // full NVLink packets) instead of 16 bytes out of every 32 as the plain mapping did.
      const size_t nblk = nv & ~(size_t)31;
      xb::batched<8, int4>(nblk, tid, nthreads,
                           [&](size_t i) {
                             const char* p = (const char*)s + (i & ~(size_t)31) * 16 + (i & 31) * 8;
                             const uint2 a = xb::ld8(p), b = xb::ld8(p + 256);
                             return make_int4((int)a.x, (int)a.y, (int)b.x, (int)b.y);
                           },
                           [&](size_t i, const int4& v) {
                             float4 lo, hi;
                             xb::unpack_bf16x8(v, &lo, &hi);
                             float* o = d + (i & ~(size_t)31) * 8 + (i & 31) * 4;
                             if (acc) {
                               xb::red_v4_f32(o, lo);
                               xb::red_v4_f32(o + 128, hi);
                             } else {
                               xb::st16f(reinterpret_cast<float4*>(o), lo);
                               xb::st16f(reinterpret_cast<float4*>(o + 128), hi);
                             }
                           });
      for (size_t i = nblk + tid; i < nv; i += nthreads) {      // the last, incomplete block: vector i = elements [8i, 8i+8)
        float4 lo, hi;
        xb::unpack_bf16x8(xb::ld16(reinterpret_cast<const int4*>(s) + i), &lo, &hi);
        if (acc) {
          xb::red_v4_f32(d + 8 * i, lo);
          xb::red_v4_f32(d + 8 * i + 4, hi);
        } else {
          xb::st16f(reinterpret_cast<float4*>(d) + 2 * i, lo);
          xb::st16f(reinterpret_cast<float4*>(d) + 2 * i + 1, hi);
        }
      }
      for (size_t i = (nv << 3) + tid; i < ne; i += nthreads) {
        float f = __bfloat162float(s[i]);
        if (acc) xb::red_f32(d + i, f); else d[i] = f;
      }
    } else {
      for (size_t i = tid; i < ne; i += nthreads) {
        float f = __bfloat162float(s[i]);
        if (acc) xb::red_f32(d + i, f); else d[i] = f;
      }
    }
    return;
  }
  if (op == OP_CAST_F32_TO_BF16) {
    size_t ne = n >> 2;
    const float* s = (const float*)src;
    __nv_bfloat16* d = (__nv_bfloat16*)dst;
    if ((((uintptr_t)s | (uintptr_t)d) & 15) == 0) {
      size_t nv = ne >> 3;   // 2 x float4 in, 8 bf16 out
      xb::batched<4, xb::F8>(nv, tid, nthreads,
                             [&](size_t i) {
                               xb::F8 r;
                               r.lo = xb::ld16f(reinterpret_cast<const float4*>(s) + 2 * i);
                               r.hi = xb::ld16f(reinterpret_cast<const float4*>(s) + 2 * i + 1);
                               return r;
                             },
                             [&](size_t i, const xb::F8& r) {
                               __nv_bfloat162 h[4];
                               h[0] = __floats2bfloat162_rn(r.lo.x, r.lo.y);
                               h[1] = __floats2bfloat162_rn(r.lo.z, r.lo.w);
                               h[2] = __floats2bfloat162_rn(r.hi.x, r.hi.y);
                               h[3] = __floats2bfloat162_rn(r.hi.z, r.hi.w);
                               int4 o;
                               memcpy(&o, h, 16);
                               xb::st16(reinterpret_cast<int4*>(d) + i, o);
                             });
      for (size_t i = (nv << 3) + tid; i < ne; i += nthreads) d[i] = __float2bfloat16_rn(s[i]);
    } else {
      for (size_t i = tid; i < ne; i += nthreads) d[i] = __float2bfloat16_rn(s[i]);
    }
    return;
  }
  if (op == OP_CAST_BF16_TO_E4M3 || op == OP_CAST_F32_TO_E4M3 || op == OP_CAST_BF16_TO_E5M2 || op == OP_CAST_F32_TO_E5M2) {
    // 8 source elements -> 8 fp8 bytes per step (one 8-byte store), saturating e4m3 / e5m2
    const bool from_bf16 = op == OP_CAST_BF16_TO_E4M3 || op == OP_CAST_BF16_TO_E5M2;
    const __nv_fp8_interpretation_t fmt = op_is_e5m2(op) ? __NV_E5M2 : __NV_E4M3;
    size_t ne = from_bf16 ? n >> 1 : n >> 2;
    unsigned char* d = (unsigned char*)dst;
    auto q1 = [&](float f) -> unsigned char {
      return (unsigned char)__nv_cvt_float_to_fp8(f * scale, __NV_SATFINITE, fmt);
    };
    auto pack8 = [&](size_t i, const xb::F8& r) {
      const float f[8] = {r.lo.x, r.lo.y, r.lo.z, r.lo.w, r.hi.x, r.hi.y, r.hi.z, r.hi.w};
      uint32_t w[2];
#pragma unroll
      for (int k = 0; k < 2; k++) {
        uint32_t a = __nv_cvt_float2_to_fp8x2(make_float2(f[4 * k] * scale, f[4 * k + 1] * scale), __NV_SATFINITE, fmt);
        uint32_t b = __nv_cvt_float2_to_fp8x2(make_float2(f[4 * k + 2] * scale, f[4 * k + 3] * scale), __NV_SATFINITE, fmt);
        w[k] = (a & 0xffffu) | (b << 16);
      }
      xb::st8(d + 8 * i, make_uint2(w[0], w[1]));
    };
    if ((((uintptr_t)src) & 15) == 0 && (((uintptr_t)d) & 7) == 0) {
      size_t nv = ne >> 3;
      if (from_bf16) {
        xb::batched<8, int4>(nv, tid, nthreads, [&](size_t i) { return xb::ld16(reinterpret_cast<const int4*>(src) + i); },
                             [&](size_t i, const int4& v) {
                               xb::F8 r;
                               xb::unpack_bf16x8(v, &r.lo, &r.hi);
                               pack8(i, r);
                             });
      } else {
        xb::batched<4, xb::F8>(nv, tid, nthreads,
                               [&](size_t i) {
                                 xb::F8 r;
                                 r.lo = xb::ld16f(reinterpret_cast<const float4*>(src) + 2 * i);
                                 r.hi = xb::ld16f(reinterpret_cast<const float4*>(src) + 2 * i + 1);
                                 return r;
                               },
                               pack8);
      }
      for (size_t i = (nv << 3) + tid; i < ne; i += nthreads)
        d[i] = q1(from_bf16 ? __bfloat162float(((const __nv_bfloat16*)src)[i]) : ((const float*)src)[i]);
    } else {
      for (size_t i = tid; i < ne; i += nthreads)
        d[i] = q1(from_bf16 ? __bfloat162float(((const __nv_bfloat16*)src)[i]) : ((const float*)src)[i]);
    }
    return;
  }
  if (op == OP_ACC_E4M3_TO_F32 || op == OP_ACC_E5M2_TO_F32 || op == OP_CAST_E4M3_TO_F32 || op == OP_CAST_E5M2_TO_F32) {
    const __nv_fp8_interpretation_t fmt = op_is_e5m2(op) ? __NV_E5M2 : __NV_E4M3;
    const bool acc = op == OP_ACC_E4M3_TO_F32 || op == OP_ACC_E5M2_TO_F32;   // else: overwrite (plain decompression)
    size_t ne = n;
    const unsigned char* s = (const unsigned char*)src;
    float* d = (float*)dst;
    auto dq = [&](unsigned char b) -> float {
      __half_raw h = __nv_cvt_fp8_to_halfraw(b, fmt);
      __half hh;
      memcpy(&hh, &h, sizeof(hh));
      return __half2float(hh) * scale;
    };
    auto put4 = [&](float* o, const unsigned char* b) {
      const float4 v = make_float4(dq(b[0]), dq(b[1]), dq(b[2]), dq(b[3]));
      if (acc) xb::red_v4_f32(o, v); else xb::st16f(reinterpret_cast<float4*>(o), v);
    };
    auto put1 = [&](float* o, unsigned char b) {
      if (acc) xb::red_f32(o, dq(b)); else *o = dq(b);
    };
    if ((((uintptr_t)s) & 7) == 0 && (((uintptr_t)d) & 15) == 0) {
      size_t nv = ne >> 3;
      // same lane interleave as the bf16 path: vector l of a 32-vector block = bytes [4l, 4l+4) and [128+4l, 128+4l+4)
      const size_t nblk = nv & ~(size_t)31;
      xb::batched<8, uint2>(nblk, tid, nthreads,
                            [&](size_t i) {
                              const unsigned char* p = s + (i & ~(size_t)31) * 8 + (i & 31) * 4;
                              uint2 r;
                              r.x = xb::ld4(p);
                              r.y = xb::ld4(p + 128);
                              return r;
                            },
                            [&](size_t i, const uint2& v) {
                              unsigned char b[8];
                              memcpy(b, &v, 8);
                              float* o = d + (i & ~(size_t)31) * 8 + (i & 31) * 4;
                              put4(o, b);
                              put4(o + 128, b + 4);
                            });
      for (size_t i = nblk + tid; i < nv; i += nthreads) {
        const uint2 v = xb::ld8(s + 8 * i);
        unsigned char b[8];
        memcpy(b, &v, 8);
        put4(d + 8 * i, b);
        put4(d + 8 * i + 4, b + 4);
      }
      for (size_t i = (nv << 3) + tid; i < ne; i += nthreads) put1(d + i, s[i]);
    } else {
      for (size_t i = tid; i < ne; i += nthreads) put1(d + i, s[i]);
    }
    return;
  }
}

}  // namespace cuda
}  // namespace bnet

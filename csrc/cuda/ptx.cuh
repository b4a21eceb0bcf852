// Inline-PTX helpers for the sm_90a kernels (memory-model loads/stores, vector
// reductions, clusters/DSMEM, mbarrier + bulk async copies, NVLS multimem).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bnet {
namespace ptx {

// ---- 16-byte streaming accesses (no L1 allocation; coherent at L2 / peer) -------------
__device__ __forceinline__ int4 ld_na_v4(const int4* p) {
  int4 r;
  asm volatile("ld.global.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void st_na_v4(int4* p, const int4& v) {
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ float4 ld_na_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p) : "memory");
  return r;
}
__device__ __forceinline__ void st_na_f4(float4* p, const float4& v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// ---- fire-and-forget reductions (no return value: one packet over NVLink) --------------
__device__ __forceinline__ void red_add_f32(float* p, float v) {
  asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" :: "l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ void red_add_v4_f32(float* p, const float4& v) {
  asm volatile("red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void red_add_v4_bf16x2(uint32_t* p, const int4& v) {
  asm volatile("red.relaxed.sys.global.add.noftz.v4.bf16x2 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ---- system-scope synchronisation ------------------------------------------------------------
__device__ __forceinline__ uint64_t ld_acquire_sys_u64(const volatile uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const volatile uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys_u32(const volatile uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys_u64(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_release_sys_add_u32(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_acq_rel_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
__device__ __forceinline__ void fence_sc_sys() { asm volatile("fence.sc.sys;" ::: "memory"); }
__device__ __forceinline__ uint64_t globaltimer() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---- thread-block clusters + distributed shared memory ------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_nctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// store a POD (size multiple of 8) into the same shared variable of CTA `rank` of this cluster
template <typename T>
__device__ __forceinline__ void st_dsmem(T* local_smem_var, uint32_t rank, const T& value) {
  static_assert(sizeof(T) % 8 == 0, "st_dsmem moves 8-byte words");
  uint32_t local = (uint32_t)__cvta_generic_to_shared(local_smem_var);
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(rank));
  const uint64_t* w = reinterpret_cast<const uint64_t*>(&value);
#pragma unroll
  for (int i = 0; i < (int)(sizeof(T) / 8); i++)
    asm volatile("st.shared::cluster.u64 [%0], %1;" :: "r"(remote + 8 * i), "l"(w[i]) : "memory");
}

// ---- mbarrier + bulk async copies (TMA engine, UBLKCP in SASS) -----------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
               :: "r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t addr = (uint32_t)__cvta_generic_to_shared(bar);
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      :: "r"(addr), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src), "r"(bytes),
                  "r"((uint32_t)__cvta_generic_to_shared(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               :: "l"(gmem_dst), "r"((uint32_t)__cvta_generic_to_shared(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---- NVLS multimem (in-switch reduction / broadcast on a multicast mapping) ------------------------
__device__ __forceinline__ float4 multimem_ld_reduce_add_f32x4(const void* mc_ptr) {
  float4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(mc_ptr) : "memory");
  return r;
}
// 8 bf16 values reduced in the switch with fp32 accumulation
__device__ __forceinline__ int4 multimem_ld_reduce_add_bf16x8(const void* mc_ptr) {
  int4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(mc_ptr) : "memory");
  return r;
}
__device__ __forceinline__ int4 multimem_ld_reduce_add_f16x8(const void* mc_ptr) {
  int4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(mc_ptr) : "memory");
  return r;
}
__device__ __forceinline__ void multimem_st_v4(void* mc_ptr, const int4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(mc_ptr), "f"(__int_as_float(v.x)), "f"(__int_as_float(v.y)), "f"(__int_as_float(v.z)),
                  "f"(__int_as_float(v.w)) : "memory");
}
__device__ __forceinline__ void multimem_red_add_u32(void* mc_ptr, uint32_t v) {
  asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" :: "l"(mc_ptr), "r"(v) : "memory");
}

}  // namespace ptx
}  // namespace bnet

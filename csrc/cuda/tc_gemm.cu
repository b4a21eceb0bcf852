// Tensor-core linear layer for sm_90a: TMA -> shared memory -> wgmma (fp32 accumulator in registers) -> fused epilogue.
//
//   D[i, j] = sum_k A[i, k] * B[j, k]        A: "lane" operand, 128 rows per tile (64 per consumer warpgroup)
//                                            B: "column" operand, BN rows per tile (the MMA N dimension)
//
// Forward: both operands are K-major bf16 matrices (a torch Linear's activation [M,K] and weight [N,K] as they are), so
// either can take either role: with a large batch x is A and w is B; with a small batch (M <= 64) the roles swap so that
// the 128 accumulator rows are filled by output features instead of 3/4 padding rows.
// Backward: dX = gY . W reduces over N and dW = gY^T . X reduces over M, so W, gY and X appear with the reduction
// dimension OUTER ("MN-major" operands).  Those are staged as [64 reduction rows x 64 MN elements] TMA boxes (one per 64
// MN elements of the tile, 8 KiB each) and handed to wgmma with the transpose bit and the MN-major form of the
// shared-memory descriptor; no transposed copy of any tensor is ever made.
//
// Persistent CTAs (one per SM once there are more tiles than SMs), 3 warpgroups, warp-specialised; the ring of
// shared-memory stages runs through tile boundaries:
//   warpgroup 0, one lane  TMA producer: per stage one [128 x 64] lane box and one [BN x 64] column box (K-major operands) or
//                          [64 x 64] boxes per 64 MN elements (MN-major operands), 128-byte swizzle, completion on the
//                          stage's `full` mbarrier; a gathered batch operand is loaded from the owning rank's tensor map
//   warpgroups 1 and 2     consumers: warpgroup c owns accumulator rows 64c .. 64c+63 of the tile (BN / 2 fp32 registers per
//                          thread).  Per stage it issues 4 wgmma.mma_async (m64 x BN x k16) and keeps one stage's group in
//                          flight: once the previous group has completed, that stage goes back to the producer through its
//                          `empty` mbarrier (one arrive per warpgroup).  After the tile's last K block each warp passes its
//                          16 x BN accumulator through a shared-memory scratch, 16 x 32 at a time, so that every thread holds
//                          16 consecutive columns of one row -> bias / ReLU -> bf16 store, or (reduce mode) fp32 adds into
//                          every rank's output — multimem.red through the NVSwitch multicast mapping or red.global per
//                          peer — or into the owner's output only (reduce-scatter).  Meanwhile the producer already fills
//                          the ring with the next tile's stages.
// The index logic (tiling, TMA coordinates, epilogue addressing) is csrc/cuda/tc_body.cuh, shared with the CPU
// emulation test; the mbarrier protocol is mirrored by tests/test_tc_pipeline_model.py.
//
// Every mbarrier wait carries a watchdog (kWatchdogNs): a pipeline that stops — a descriptor the hardware rejects, a
// lost TMA completion — sets *err and lets every role fall through to the teardown instead of hanging the GPU.
// ops/tc_linear.py and ops/tc_conv.py trust the kernels only after a self-check in a child process on the GPU at hand.
// Descriptor packing is unit-tested against CuTe (csrc/tests/tc_desc_test.cc).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include <mutex>
#include <string>

#include "bnet/bnet_tc.h"
#include "cuda/driver_api.h"
#include "cuda/ptx.cuh"
#include "cuda/tc_body.cuh"

#define BNET_API extern "C" __attribute__((visibility("default")))

namespace {

using namespace bnet;
using namespace bnet::tc;              // tile constants, TcArgs, plan / setup, per-tile index logic (tc_body.cuh)

constexpr int kThreads = 384;          // producer warpgroup + two consumer warpgroups
constexpr uint64_t kWatchdogNs = 2000000000ull;

thread_local std::string g_err;

// ------------------------------------------------------------------------------------------------ descriptors
// Shared-memory matrix descriptor of wgmma (bit positions: cute/arch/mma_sm90_desc.hpp `GmmaDescriptor`):
//   [0,14) start address >> 4   [16,30) leading byte offset >> 4   [32,46) stride byte offset >> 4   [49,52) base offset
//   [62,64) layout (1 = 128-byte swizzle)
// K-major tile whose rows are 128 bytes, stored densely and swizzled by the hardware in 8-row x 128-byte atoms (what TMA
// writes with CU_TENSOR_MAP_SWIZZLE_128B): leading byte offset unused (1 like CuTe), stride byte offset = 1024 B between
// 8-row groups.  Every stage starts on a 1024-byte boundary, so the base offset is 0.
__host__ __device__ constexpr uint64_t smem_desc_sw128(uint32_t smem_addr) {
  return uint64_t((smem_addr >> 4) & 0x3FFF) | (uint64_t(1) << 16) | (uint64_t(1024 >> 4) << 32) | (uint64_t(1) << 62);
}

// The same for an MN-major tile staged as [64 reduction rows x 128 bytes] boxes, one per 64 MN elements, 8 KiB apart:
//   leading byte offset = 8192 B between 64-element MN atoms, stride byte offset = 1024 B between 8-row reduction groups
//   (CuTe: make_gmma_desc<Major::MN> of tile_to_shape(Layout_MN_SW128_Atom<bf16>, (MN, 64), Step<_2,_1>) -> LBO 512, SBO 64).
// One K = 16 slice is two 8-row groups further: +2048 B.
__host__ __device__ constexpr uint64_t smem_desc_sw128_mn(uint32_t smem_addr) {
  return uint64_t((smem_addr >> 4) & 0x3FFF) | (uint64_t(8192 >> 4) << 16) | (uint64_t(1024 >> 4) << 32) | (uint64_t(1) << 62);
}

// ------------------------------------------------------------------------------------------------ PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
// false = the watchdog fired (and *err now says which role gave up)
__device__ __forceinline__ bool mbar_wait_wd(uint32_t bar, uint32_t parity, int* err, int role) {
  if (mbar_try_wait(bar, parity)) return true;
  const uint64_t t0 = ptx::globaltimer();
  while (!mbar_try_wait(bar, parity)) {
    if (ptx::globaltimer() - t0 > kWatchdogNs) {
      atomicCAS(err, 0, role);
      return false;
    }
  }
  return true;
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      :: "r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      :: "r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" :: "l"(map) : "memory");
}
// wgmma ordering: fence before the first MMA that touches registers written by ordinary instructions; commit the MMAs
// issued so far as one group; wait until at most N groups are pending
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i]) :: "memory");
}
// true when any of the `count` threads arriving at named barrier `id` passes true
__device__ __forceinline__ bool bar_any(int id, int count, bool v) {
  uint32_t r;
  asm volatile(
      "{\n\t.reg .pred p, q;\n\t"
      "setp.ne.u32 p, %1, 0;\n\t"
      "bar.red.or.pred q, %2, %3, p;\n\t"
      "selp.u32 %0, 1, 0, q;\n\t}"
      : "=r"(r) : "r"(uint32_t(v)), "r"(id), "r"(count) : "memory");
  return r != 0;
}
// split-K fix-up: wait until `*turn` (the slices that have added their partial tile so far) reaches `mine`
__device__ __forceinline__ void wait_turn(const int* turn, int mine, int* err) {
  const uint64_t t0 = ptx::globaltimer();
  while ((int)ptx::ld_acquire_sys_u32(reinterpret_cast<const volatile uint32_t*>(turn)) != mine) {
    if (ptx::globaltimer() - t0 > kWatchdogNs) {
      atomicCAS(err, 0, 3);
      return;
    }
  }
}
__device__ __forceinline__ void multimem_red_add_f32(float* mc, float v) {
  asm volatile("multimem.red.relaxed.sys.global.add.f32 [%0], %1;" :: "l"(mc), "f"(v) : "memory");
}
__device__ __forceinline__ void multimem_red_add_v4_f32(float* mc, const float4& v) {
  asm volatile("multimem.red.relaxed.sys.global.add.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// D (m64 x N, fp32, the warpgroup's registers) (+)= A[smem] * B[smem]^T; TA / TB = 1: the operand is MN-major (transposed).
// Register d[4 j + e] of thread (warp w, lane l) holds D[16 w + l / 4 + 8 (e / 2), 8 j + 2 (l % 4) + e % 2].
template <int N, int TA, int TB>
struct Wgmma;
template <int TA, int TB>
struct Wgmma<32, TA, TB> {
  __device__ __forceinline__ static void mma(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
  }
};
template <int TA, int TB>
struct Wgmma<64, TA, TB> {
  __device__ __forceinline__ static void mma(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
  }
};
template <int TA, int TB>
struct Wgmma<128, TA, TB> {
  __device__ __forceinline__ static void mma(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
  }
};
template <int TA, int TB>
struct Wgmma<256, TA, TB> {
  __device__ __forceinline__ static void mma(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
  }
};

// ------------------------------------------------------------------------------------------------ kernel
// the epilogue's memory operations (tc_body.cuh::epilogue_chunk)
struct DeviceOut {
  __device__ __forceinline__ void st16(uint16_t* p, uint16_t v) const { *p = v; }
  __device__ __forceinline__ void st16x16(uint16_t* row, const float (&f)[16]) const {
    uint32_t w[8];
#pragma unroll
    for (int u = 0; u < 8; u++) {
      __nv_bfloat162 p = __floats2bfloat162_rn(f[2 * u], f[2 * u + 1]);
      w[u] = *reinterpret_cast<uint32_t*>(&p);
    }
    reinterpret_cast<uint4*>(row)[0] = make_uint4(w[0], w[1], w[2], w[3]);
    reinterpret_cast<uint4*>(row)[1] = make_uint4(w[4], w[5], w[6], w[7]);
  }
  __device__ __forceinline__ void add1(float* p, float v, bool multicast) const {
    if (multicast) multimem_red_add_f32(p, v); else ptx::red_add_f32(p, v);
  }
  __device__ __forceinline__ void add4(float* p, const float* f, bool multicast) const {
    const float4 x = make_float4(f[0], f[1], f[2], f[3]);
    if (multicast) multimem_red_add_v4_f32(p, x); else ptx::red_add_v4_f32(p, x);
  }
};

// the batch operand's tensor maps: one, or one per rank when its row blocks live on different GPUs
struct TcBatchMaps { CUtensorMap m[BNET_TC_MAX_PEERS]; };

template <int BN>
struct Smem {
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
};

// kSwap:   false -> A = x (lane i = batch row m), B = w (column j = feature n); out[m, n] = out[i * ldo + j]
//          true  -> A = w (lane i = feature n),   B = x (column j = batch row m); out[m, n] = out[j * ldo + i]
// kReduce: fp32 adds into args.outs[] instead of a bf16 store
//
// Persistent over output tiles: CTA c takes tiles c, c + gridDim.x, ... (consecutive CTAs share the column operand's
// block, so it is read from HBM once and from L2 afterwards).  The shared-memory ring runs straight through tile
// boundaries: while the consumers run a tile's epilogue, the producer fills the stages of the next tile.  With
// gridDim.x == n_tiles every CTA simply does one tile.
// kAMn / kBMn: the lane / column operand is MN-major (reduction dimension outer) instead of K-major
// kConv: 1 = the lane operand is a 3x3 convolution's input patch, loaded as 4-D TMA boxes (tc_body.cuh::ConvGeom);
//        2 = convolution weight gradient: BOTH operands are 4-D boxes of NHWC activations (gy on the lanes through
//            maps_batch.m[0], the shifted input on the columns through map_feat), MN-major, the reduction runs over pixels
template <int BN, int kStages, bool kSwap, bool kReduce, bool kAMn, bool kBMn, int kConv = 0>
__global__ void __launch_bounds__(kThreads, 1)
tc_linear_kernel(const __grid_constant__ TcBatchMaps maps_batch, const __grid_constant__ CUtensorMap map_feat, const TcArgs args) {
  static_assert(BN % 32 == 0 && BN >= 32 && BN <= 256, "wgmma N, in whole 32-column epilogue chunks");
  static_assert(!kBMn || BN % 64 == 0, "an MN-major operand is staged in 64-element atoms");
  static_assert(kConv != 1 || (!kSwap && !kAMn && !kReduce), "convolution: pixels ride the lanes, K-major patches, bf16 store");
  static_assert(kConv != 2 || (!kSwap && kAMn && kBMn && kReduce), "weight gradient: MN-major operands, split over pixel blocks");
  extern __shared__ uint8_t smem_raw[];
  // swizzle-128B atoms must start on 1024-byte boundaries of the shared window
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* const tiles = smem_raw + (base - raw);
  float* const scratch = reinterpret_cast<float*>(tiles + kStages * Smem<BN>::kStageBytes);
  uint64_t* const bars = reinterpret_cast<uint64_t*>(scratch + kEpiScratchBytes / 4);
  const uint32_t full0 = smem_u32(bars), empty0 = full0 + 8 * kStages;
  uint32_t* const last_slot = reinterpret_cast<uint32_t*>(bars + 2 * kStages);   // split-K fix-up: "this CTA's slice was last"
  uint32_t* const pos_slot = last_slot + 1;                                       // this CTA's (x, z) position, z * gridDim.x + x

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool fix = kReduce && args.fix_out != nullptr;

  if (warp == 0 && lane == 0) {
    if (fix) {
      // serial split-K (slice z adds after slices 0 .. z-1, below): positions are handed out in the order the CTAs START, so a
      // slice only ever waits for slices whose CTAs already run or are done, however the hardware dispatches the grid.  The
      // ticket is the int after the tile counters; the CTA that takes the last one puts it back to 0 for the next launch.
      uint32_t* ticket = reinterpret_cast<uint32_t*>(args.fix_counters + args.n_tiles);
      const uint32_t v = atomicAdd(ticket, 1u);
      if (v == gridDim.x * gridDim.z - 1) atomicExch(ticket, 0u);
      *pos_slot = v;
    } else {
      *pos_slot = blockIdx.z * gridDim.x + blockIdx.x;
    }
    tma_prefetch_desc(&maps_batch.m[0]);
    tma_prefetch_desc(&map_feat);
    for (int s = 0; s < kStages; s++) {
      ptx::mbar_init(bars + s, 1);               // full: the producer's arrive.expect_tx (+ TMA bytes)
      ptx::mbar_init(bars + kStages + s, 2);     // empty: one arrive per consumer warpgroup
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  const int bx = (int)(*pos_slot % gridDim.x), bz = (int)(*pos_slot / gridDim.x);
  const int kb_begin = bz * args.k_per_split;
  const int kb_end = min(kb_begin + args.k_per_split, args.k_blocks);
  const int nkb = kb_end - kb_begin;       // >= 1 by construction of the grid

  // the producer warpgroup needs few registers, a consumer holds BN / 2 accumulators: hand the register file over
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 0 && lane == 0) {
      uint32_t g = 0;                              // k-blocks issued by this CTA so far (ring position)
      bool alive = true;
      for (int t = bx; t < args.n_tiles && alive; t += gridDim.x) {
        // the operand that is the batch rides the lanes (plain) or the columns (swapped); when it is gathered, the tile's
        // rows come from ONE rank's map, at a row offset inside that rank's shard (tc_body.cuh::tile_coord)
        const TileCoord tc = tile_coord<BN, kSwap>(args, t);
        const CUtensorMap* map_a = kSwap ? &map_feat : &maps_batch.m[tc.a_map];
        const CUtensorMap* map_b = kSwap ? &maps_batch.m[tc.b_map] : &map_feat;
        ConvTile ct{};
        if constexpr (kConv == 1) ct = conv_tile<BN>(args, t);
        for (int i = 0; i < nkb; i++, g++) {
          const uint32_t s = g % kStages, round = g / kStages;
          if (round > 0 && !mbar_wait_wd(empty0 + 8 * s, (round - 1) & 1, args.err, 1)) { alive = false; break; }
          const uint32_t a_dst = base + s * Smem<BN>::kStageBytes, bar = full0 + 8 * s;
          mbar_expect_tx(bar, Smem<BN>::kStageBytes);
          if constexpr (kConv == 1) {
            conv_stage_loads<BN, kBMn>(args, ct, kb_begin + i,
                [&](int offset, int c0, int c1, int c2, int c3) { tma_load_4d(a_dst + offset, &maps_batch.m[0], bar, c0, c1, c2, c3); },
                [&](int offset, int c0, int c1) { tma_load_2d(a_dst + kABytes + offset, &map_feat, bar, c0, c1); });
          } else if constexpr (kConv == 2) {
            wgrad_stage_loads<BN>(args, tc, kb_begin + i,
                [&](int offset, int c0, int c1, int c2, int c3) { tma_load_4d(a_dst + offset, &maps_batch.m[0], bar, c0, c1, c2, c3); },
                [&](int offset, int c0, int c1, int c2, int c3) { tma_load_4d(a_dst + kABytes + offset, &map_feat, bar, c0, c1, c2, c3); });
          } else {
            stage_loads<BN, kAMn, kBMn>(tc, (kb_begin + i) * kBK, [&](int operand, int offset, int c0, int c1) {
              tma_load_2d(a_dst + (operand ? kABytes : 0) + offset, operand ? map_b : map_a, bar, c0, c1);
            });
          }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    // ---- consumers: warpgroup c = accumulator rows 64c .. 64c+63; warp wq of it = rows 16 wq .. 16 wq + 15 of those
    const int c = (warp >> 2) - 1, wq = warp & 3;
    const int ctid = threadIdx.x - 128;            // 0 .. 255 over both consumer warpgroups
    const bool signal = (warp & 3) == 0 && lane == 0;
    // descriptor advance per K = 16 slice, in 16-byte units: 32 B along the swizzled row (K-major), or two 8-row groups
    // = 2048 B (MN-major).  Warpgroup c's half of the lane operand starts 64 rows (K-major) or one 64-element atom
    // (MN-major) further — 8 KiB either way.
    constexpr uint64_t kStepA = kAMn ? 2048 / 16 : kMmaK * 2 / 16, kStepB = kBMn ? 2048 / 16 : kMmaK * 2 / 16;
    float* const scr = scratch + (warp - 4) * (16 * kEpiPitch);
    const bool add_bias = args.bias != nullptr && (!kReduce || bz == 0) && !fix;
    float acc[BN / 2];
    uint32_t g = 0;
    bool alive = true;
    for (int t = bx; t < args.n_tiles; t += gridDim.x) {
      for (int i = 0; i < nkb; i++, g++) {
        const uint32_t s = g % kStages;
        alive = mbar_wait_wd(full0 + 8 * s, (g / kStages) & 1, args.err, 2);
        if (!alive) break;
        const uint32_t a_src = base + s * Smem<BN>::kStageBytes;
        const uint64_t da = kAMn ? smem_desc_sw128_mn(a_src + c * 8192) : smem_desc_sw128(a_src + c * 8192);
        const uint64_t db = kBMn ? smem_desc_sw128_mn(a_src + kABytes) : smem_desc_sw128(a_src + kABytes);
        wgmma_fence();
        fence_regs(acc);
#pragma unroll
        for (int k = 0; k < kBK / kMmaK; k++)
          Wgmma<BN, kAMn, kBMn>::mma(acc, da + uint64_t(k) * kStepA, db + uint64_t(k) * kStepB, (i | k) != 0 ? 1u : 0u);
        wgmma_commit();
        fence_regs(acc);
        if (i > 0) {
          wgmma_wait<1>();                           // the previous stage's MMAs have read their operands
          if (signal) mbar_arrive(empty0 + 8 * ((g - 1) % kStages));
        }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (alive && signal) mbar_arrive(empty0 + 8 * ((g - 1) % kStages));
      // both warpgroups agree before anything that synchronises them (the fix-up below) can wait for a quitter
      if (bar_any(1, 256, !alive)) break;

      TileCoord tc = tile_coord<BN, kSwap>(args, t);
      ConvTile ct{};
      if constexpr (kConv == 1) {
        ct = conv_tile<BN>(args, t);
        tc.b_row0 = ct.b_row0;
      }
      // ---- epilogue, 32 accumulator columns at a time: the warp's fragment goes to its scratch (row pitch kEpiPitch
      //      floats keeps the float2 stores free of bank conflicts), then lane l takes row l % 16,
      //      columns 16 (l / 16) .. +15
      const int r_own = lane & 15, h_own = lane >> 4;
      const int i_local = 64 * c + 16 * wq + r_own;     // row of the tile this thread finishes
      int i_glob = tc.a_row0 + i_local;
      if constexpr (kConv == 1) {
        // the row is a pixel of the tile's patch: its row in the [N*H*W, Cout] output, or "past the end" outside the image
        const long long row = conv_out_row(args, ct, i_local);
        i_glob = row < 0 ? args.rows_a : (int)row;
      }
      if constexpr (kReduce) {
        if (fix) {
          // serial split-K: slice z adds its partial tile only after slices 0 .. z-1 have added theirs, so every element is
          // summed in the same order on every run (the counter is the one the fix-up below advances)
          if (ctid == 0) wait_turn(args.fix_counters + t, bz, args.err);
          asm volatile("bar.sync 1, 256;" ::: "memory");
        }
      }
#pragma unroll
      for (int cc = 0; cc < BN / 32; cc++) {
        __syncwarp();
#pragma unroll
        for (int jj = 0; jj < 4; jj++) {
          const int j = 4 * cc + jj, col = 8 * jj + 2 * (lane & 3), row = lane >> 2;
          *reinterpret_cast<float2*>(scr + row * kEpiPitch + col) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(scr + (row + 8) * kEpiPitch + col) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        __syncwarp();
        float v[16];
#pragma unroll
        for (int u = 0; u < 16; u += 4) {
          const float4 x = *reinterpret_cast<const float4*>(scr + r_own * kEpiPitch + 16 * h_own + u);
          v[u] = x.x; v[u + 1] = x.y; v[u + 2] = x.z; v[u + 3] = x.w;
        }
        epilogue_chunk<kSwap, kReduce>(args, i_glob, tc.b_row0 + 32 * cc + 16 * h_own, v, add_bias, DeviceOut{});
      }
      if constexpr (kReduce) {
        if (fix) {
          // ---- split-K fix-up: the last K slice to arrive finishes the tile (see TcArgs::fix_out)
          __threadfence();                                                   // this thread's adds, device-wide
          asm volatile("bar.sync 1, 256;" ::: "memory");                     // ... and those of all 256 consumer threads
          if (ctid == 0) *last_slot = (atomicAdd(args.fix_counters + t, 1) == (int)gridDim.z - 1) ? 1u : 0u;
          asm volatile("bar.sync 1, 256;" ::: "memory");
          if (*(volatile uint32_t*)last_slot) {
            __threadfence();
            TcArgs fa = args;
            fa.outs[0] = args.fix_out;
            fa.ldo = args.fix_ldo;
            float* ws = static_cast<float*>(args.outs[0]);
            // thread -> (tile row ctid % 128, column half ctid / 128)
            const int fi = tc.a_row0 + (ctid & 127);
            if (fi < args.rows_a) {
#pragma unroll 1
              for (int q = 0; q < BN / 32; q++) {
                const int j0 = tc.b_row0 + (ctid >> 7) * (BN / 2) + q * 16;
                if (j0 >= args.rows_b) break;
                float v[16];
#pragma unroll
                for (int u = 0; u < 16; u++) {
                  v[u] = 0.f;
                  if (j0 + u < args.rows_b) {
                    float* p = kSwap ? ws + size_t(j0 + u) * args.ldo + fi : ws + size_t(fi) * args.ldo + j0 + u;
                    v[u] = __ldcg(p);
                    __stcg(p, 0.f);                                           // the workspace is clean for the next call
                  }
                }
                epilogue_chunk<kSwap, false>(fa, fi, j0, v, args.bias != nullptr, DeviceOut{});
              }
            }
            if (ctid == 0) args.fix_counters[t] = 0;
          }
          asm volatile("bar.sync 1, 256;" ::: "memory");                     // last_slot is reused by the next tile
        }
      }
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    else
      (void)cudaGetLastError();
  });
  return fn;
}

// MapDesc (tc_body.cuh) -> CUtensorMap: 2-D bf16, boxes of [box1 x box0], 128-byte swizzle; rows / columns outside the
// matrix read as zero, so ragged extents need no special case in the kernel
bool make_map(CUtensorMap* map, const MapDesc& d) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) { g_err = "the CUDA driver does not export cuTensorMapEncodeTiled"; return false; }
  if ((reinterpret_cast<uintptr_t>(d.ptr) & 15) || (size_t(d.pitch_elems) * 2) % 16) {
    g_err = "operands must be 16-byte aligned with a row pitch that is a multiple of 8 elements";
    return false;
  }
  const cuuint64_t dims[2] = {cuuint64_t(d.dim0), cuuint64_t(d.dim1)};
  const cuuint64_t strides[1] = {cuuint64_t(d.pitch_elems) * 2};
  const cuuint32_t box[2] = {cuuint32_t(d.box0), cuuint32_t(d.box1)};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(d.ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { g_err = "cuTensorMapEncodeTiled failed: " + std::to_string(int(r)); return false; }
  return true;
}

template <int BN, int kStages, bool kSwap, bool kReduce, bool kAMn, bool kBMn, int kConv = 0>
int launch(const TcBatchMaps& mbatch, const CUtensorMap& mfeat, const TcArgs& a, const BnetTcPlan& p, cudaStream_t st) {
  auto kern = tc_linear_kernel<BN, kStages, kSwap, kReduce, kAMn, kBMn, kConv>;
  static std::once_flag once;
  static cudaError_t attr_rc = cudaSuccess;
  const int smem = p.smem_bytes;
  std::call_once(once, [&] { attr_rc = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); });
  if (attr_rc != cudaSuccess) { g_err = std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(attr_rc); return -1; }
  kern<<<dim3(p.ctas, 1, p.grid_z), kThreads, smem, st>>>(mbatch, mfeat, a);
  cudaError_t rc = cudaGetLastError();
  if (rc != cudaSuccess) { g_err = std::string("tc_linear launch: ") + cudaGetErrorString(rc); return -1; }
  return 1;
}

// SMs of the current device; 132 (H100 SXM) when there is none to ask (host-only planning in the CPU tests)
int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0)
      n = v;
    else { (void)cudaGetLastError(); n = 132; }
  }
  return n;
}

// `batch` / `feat`: the two operands in problem order (out[batch index, feature index]); the plan decides which of them
// rides the accumulator rows.  bias is indexed by the feature.  All the index logic is tc_body.cuh::setup_problem (pure, unit-
// tested on the CPU); here the map descriptions are encoded and the instantiation is picked.
int run(const Operand& batch, const Operand& feat, int red, const void* bias, void* const* outs, int n_outs, int multicast,
        bool reduce, int ldo, int act, int splits, int* err_dev, void* stream, const void* const* shards = nullptr,
        int n_shards = 0, int scatter_ranks = 0, void* fix_out = nullptr, int* fix_counters = nullptr, int fix_ldo = 0) {
  Problem pr;
  if (const char* e = setup_problem(batch, feat, red, bias, outs, n_outs, multicast, reduce, ldo, act, splits, err_dev, shards,
                                    n_shards, scatter_ranks, sm_count(), &pr)) {
    g_err = e;
    return -1;
  }
  pr.args.fix_out = fix_out;
  pr.args.fix_counters = fix_counters;
  pr.args.fix_ldo = fix_ldo;
  TcBatchMaps mbatch;
  CUtensorMap mfeat;
  for (int r = 0; r < pr.n_batch_maps; r++)
    if (!make_map(&mbatch.m[r], pr.batch_maps[r])) return -1;
  if (!make_map(&mfeat, pr.feat_map)) return -1;
  const BnetTcPlan& p = pr.plan;
  const TcArgs& a = pr.args;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool amn = pr.a_mn, bmn = pr.b_mn, swap = p.swap != 0;
#define BNET_TC_CASE(BN, SWAP, RED, AMN, BMN)                                          \
  if (p.bn == BN && swap == SWAP && reduce == RED && amn == AMN && bmn == BMN)        \
    return launch<BN, stages_for(BN), SWAP, RED, AMN, BMN>(mbatch, mfeat, a, p, st);
  // forward (K-major x K-major), plain and with the cross-rank adds
  BNET_TC_CASE(32, true, false, false, false)   BNET_TC_CASE(32, true, true, false, false)
  BNET_TC_CASE(64, true, false, false, false)   BNET_TC_CASE(64, true, true, false, false)
  BNET_TC_CASE(128, false, false, false, false) BNET_TC_CASE(128, false, true, false, false)
  BNET_TC_CASE(256, false, false, false, false) BNET_TC_CASE(256, false, true, false, false)
  // dX = gY . W: gY K-major; W MN-major — on the columns (large batch) or on the lanes (small batch)
  BNET_TC_CASE(128, false, false, false, true)  BNET_TC_CASE(256, false, false, false, true)
  BNET_TC_CASE(32, true, false, true, false)    BNET_TC_CASE(64, true, false, true, false)
  // dW = gY^T . X: both MN-major
  BNET_TC_CASE(128, false, false, true, true)   BNET_TC_CASE(256, false, false, true, true)
#undef BNET_TC_CASE
  g_err = "no kernel for this plan";
  return -1;
}


// 4-D map over an NHWC activation {C, W, H, N}: boxes of {64 channels, bw, bh, bn}, 128-byte swizzle, zero fill
bool make_map_nhwc(CUtensorMap* map, const MapDesc4& d) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) { g_err = "the CUDA driver does not export cuTensorMapEncodeTiled"; return false; }
  if ((reinterpret_cast<uintptr_t>(d.ptr) & 15) || d.C % 8) { g_err = "activations must be 16-byte aligned with C a multiple of 8"; return false; }
  const cuuint64_t dims[4] = {cuuint64_t(d.C), cuuint64_t(d.W), cuuint64_t(d.H), cuuint64_t(d.N)};
  const cuuint64_t strides[3] = {cuuint64_t(d.C) * 2, cuuint64_t(d.W) * d.C * 2, cuuint64_t(d.H) * d.W * d.C * 2};
  const cuuint32_t box[4] = {cuuint32_t(kBK), cuuint32_t(d.bw), cuuint32_t(d.bh), cuuint32_t(d.bn)};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(d.ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { g_err = "cuTensorMapEncodeTiled (NHWC) failed: " + std::to_string(int(r)); return false; }
  return true;
}

// the index logic is tc_body.cuh::setup_conv (pure, emulated on the CPU by tc_emu_test); here the maps are encoded and the
// instantiation is picked
int run_conv(const void* x, const void* w, const void* bias, void* out, int N, int H, int W, int Cred, int Cn, int act, int dgrad,
             int* err_dev, void* stream) {
  ConvProblem cp;
  if (const char* e = setup_conv(x, w, bias, out, N, H, W, Cred, Cn, act, dgrad, err_dev, sm_count(), &cp)) {
    g_err = e;
    return -1;
  }
  TcBatchMaps mbatch;
  CUtensorMap mfeat;
  if (!make_map_nhwc(&mbatch.m[0], cp.x_map)) return -1;
  if (!make_map(&mfeat, cp.w_map)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const BnetTcPlan& p = cp.plan;
#define BNET_CONV_CASE(BN, BMN) \
  if (p.bn == BN && cp.dgrad == BMN) return launch<BN, stages_for(BN), false, false, false, BMN, 1>(mbatch, mfeat, cp.args, p, st);
  BNET_CONV_CASE(64, false) BNET_CONV_CASE(128, false) BNET_CONV_CASE(256, false)
  BNET_CONV_CASE(64, true)  BNET_CONV_CASE(128, true)  BNET_CONV_CASE(256, true)
#undef BNET_CONV_CASE
  g_err = "no convolution kernel for this plan";
  return -1;
}

// filter gradient: index logic tc_body.cuh::setup_conv_wgrad; both tensor maps are 4-D NHWC maps with 64-pixel boxes
int run_conv_wgrad(const void* gy, const void* x, void* dw, float* ws, int* counters, int N, int H, int W, int Cin, int Cout, int splits,
                   int* err_dev, void* stream) {
  WgradProblem wp;
  // BNET_TC_WGRAD_BN=128: every layer on 128-column tiles (ops/tc_conv.py sets it when only that configuration passed the
  // self-check on the GPU at hand)
  // BNET_TC_WGRAD_FIXUP=0: the slices only add into the fp32 workspace, the caller converts and clears it (ops/tc_conv.py)
  static const int force_bn = [] { const char* v = getenv("BNET_TC_WGRAD_BN"); return v ? atoi(v) : 0; }();
  static const int fixup = [] { const char* v = getenv("BNET_TC_WGRAD_FIXUP"); return v ? atoi(v) : 1; }();
  if (const char* e = setup_conv_wgrad(gy, x, ws, dw, counters, N, H, W, Cin, Cout, splits, err_dev, sm_count(), &wp, force_bn, fixup)) {
    g_err = e;
    return -1;
  }
  if (reinterpret_cast<uintptr_t>(dw) & 15) { g_err = "the filter gradient must be 16-byte aligned"; return -1; }
  TcBatchMaps mbatch;
  CUtensorMap mfeat;
  if (!make_map_nhwc(&mbatch.m[0], wp.gy_map)) return -1;
  if (!make_map_nhwc(&mfeat, wp.x_map)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const BnetTcPlan& p = wp.plan;
  if (p.bn == 128) return launch<128, stages_for(128), false, true, true, true, 2>(mbatch, mfeat, wp.args, p, st);
  if (p.bn == 256) return launch<256, stages_for(256), false, true, true, true, 2>(mbatch, mfeat, wp.args, p, st);
  g_err = "no weight-gradient kernel for this plan";
  return -1;
}

}  // namespace

BNET_API const char* bnet_tc_last_error(void) { return g_err.c_str(); }
BNET_API uint64_t bnet_tc_smem_desc(uint32_t smem_addr) { return smem_desc_sw128(smem_addr); }
BNET_API uint64_t bnet_tc_smem_desc_mn(uint32_t smem_addr) { return smem_desc_sw128_mn(smem_addr); }

BNET_API int bnet_tc_supported(void) {
  int dev = 0, major = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  return (major == 9 && encode_fn() != nullptr) ? 1 : 0;
}

BNET_API int bnet_tc_plan(int M, int N, int K, int reduce, int splits, BnetTcPlan* p) {
  if (!p || M < 1 || N < 1 || K < 1) { g_err = "bad problem size"; return -1; }
  if (K % 8) { g_err = "K must be a multiple of 8 (16-byte TMA row pitch)"; return -1; }
  if (plan_gemm(M, N, K, reduce, splits, sm_count(), p) != 0) { g_err = "problem too large for one launch"; return -1; }
  return 0;
}

BNET_API int bnet_tc_linear(const void* x, const void* w, const void* bias, void* out, int M, int N, int K, int ldx, int ldw,
                            int ldo, int act, int* err_dev, void* stream) {
  void* outs[1] = {out};
  return run(Operand{x, M, ldx, 0}, Operand{w, N, ldw, 0}, K, bias, outs, 1, 0, false, ldo, act, 1, err_dev, stream);
}

BNET_API int bnet_tc_linear_reduce(const void* x, const void* w, const void* bias, void* const* outs, int n_outs, int multicast,
                                   int M, int N, int K, int ldx, int ldw, int ldo, int splits, int* err_dev, void* stream) {
  return run(Operand{x, M, ldx, 0}, Operand{w, N, ldw, 0}, K, bias, outs, n_outs, multicast, true, ldo, BNET_TC_ACT_NONE, splits,
             err_dev, stream);
}

// Split-K with the finish inside the kernel: `ws` is an fp32 [M, N] workspace and `counters` one int per output tile
// (bnet_tc_plan: grid_x * grid_y) plus one, BOTH all zero on entry — the kernel leaves them all zero again, so they are allocated
// and cleared once.  out = act(x . w^T + bias) in bf16, one launch.
BNET_API int bnet_tc_linear_splitk(const void* x, const void* w, const void* bias, void* out, float* ws, int* counters, int M, int N,
                                   int K, int ldx, int ldw, int ldo, int act, int splits, int* err_dev, void* stream) {
  void* outs[1] = {ws};
  if (!ws || !counters) { g_err = "split-K needs a workspace and tile counters"; return -1; }
  return run(Operand{x, M, ldx, 0}, Operand{w, N, ldw, 0}, K, bias, outs, 1, 0, true, N, act, splits, err_dev, stream, nullptr, 0, 0,
             out, counters, ldo);
}

// dx[M, K] = gy[M, N] . w[N, K]: the reduction runs over N, so w is read with its rows as the reduction (MN-major)
BNET_API int bnet_tc_linear_dgrad(const void* gy, const void* w, void* dx, int M, int N, int K, int ldgy, int ldw, int lddx,
                                  int* err_dev, void* stream) {
  void* outs[1] = {dx};
  return run(Operand{gy, M, ldgy, 0}, Operand{w, K, ldw, 1}, N, nullptr, outs, 1, 0, false, lddx, BNET_TC_ACT_NONE, 1, err_dev,
             stream);
}

// dw[N, K] = gy[M, N]^T . x[M, K]: the reduction runs over the batch; both operands are MN-major.  dw's two extents are
// feature counts, so the plan never swaps when N > 64 (and a layer with <= 64 outputs simply takes the swapped tiles).
BNET_API int bnet_tc_linear_wgrad(const void* gy, const void* x, void* dw, int M, int N, int K, int ldgy, int ldx, int lddw,
                                  int* err_dev, void* stream) {
  void* outs[1] = {dw};
  if (N <= 64) { g_err = "wgrad needs more than 64 output features (use cuBLAS for tiny layers)"; return -1; }
  return run(Operand{gy, N, ldgy, 1}, Operand{x, K, ldx, 1}, M, nullptr, outs, 1, 0, false, lddw, BNET_TC_ACT_NONE, 1, err_dev,
             stream);
}

// out[n_shards * rows_per_shard, N] = act([x_0; x_1; ...] . w^T + bias): the all-gather of a sequence/batch-sharded
// activation fused into the GEMM's operand loads — shard r is read straight from x_shards[r] (rank r's symmetric heap,
// mapped over NVLink) by TMA, tile by tile, while the tensor cores work on the previous tile.
BNET_API int bnet_tc_allgather_linear(const void* const* x_shards, int n_shards, int rows_per_shard, const void* w, const void* bias,
                                      void* out, int N, int K, int ldx, int ldw, int ldo, int act, int* err_dev, void* stream) {
  void* outs[1] = {out};
  if (n_shards < 1 || rows_per_shard < 1) { g_err = "bad shard arguments"; return -1; }
  return run(Operand{x_shards[0], n_shards * rows_per_shard, ldx, 0}, Operand{w, N, ldw, 0}, K, bias, outs, 1, 0, false, ldo, act, 1,
             err_dev, stream, x_shards, n_shards, 0);
}

// outs[r][M / n_ranks, N] += rows [r * M / n_ranks, (r + 1) * M / n_ranks) of x . w^T: GEMM + reduce-scatter in one kernel
// (every rank calls it with its K-shard; each output tile travels once, to its owner).
BNET_API int bnet_tc_linear_reduce_scatter(const void* x, const void* w, const void* bias, void* const* outs, int n_ranks, int M,
                                           int N, int K, int ldx, int ldw, int ldo, int splits, int* err_dev, void* stream) {
  return run(Operand{x, M, ldx, 0}, Operand{w, N, ldw, 0}, K, bias, outs, n_ranks, 0, true, ldo, BNET_TC_ACT_NONE, splits, err_dev,
             stream, nullptr, 0, n_ranks);
}

// 3x3 / stride 1 / pad 1 convolution on the same kernel (implicit GEMM: 4-D TMA boxes of the NHWC activation, the padding
// is the TMA unit's zero fill), bias and ReLU in the epilogue.  bf16 NHWC in and out, filters as torch stores a
// channels_last Conv2d weight ([Cout][3][3][Cin]).  Cin must be a multiple of 64, Cout of 8.
BNET_API int bnet_tc_conv3x3(const void* x, const void* w, const void* bias, void* out, int N, int H, int W, int Cin, int Cout,
                             int act, int* err_dev, void* stream) {
  return run_conv(x, w, bias, out, N, H, W, Cin, Cout, act, 0, err_dev, stream);
}
// dx[N,H,W,Cin] = conv3x3 of gy[N,H,W,Cout] with the same filter w[Cout][3][3][Cin], taps flipped, filter read MN-major
// (no transposed / rotated copy of the filter is made).  Cout and Cin must be multiples of 64.
BNET_API int bnet_tc_conv3x3_dgrad(const void* gy, const void* w, void* dx, int N, int H, int W, int Cin, int Cout, int* err_dev,
                                   void* stream) {
  return run_conv(gy, w, nullptr, dx, N, H, W, Cout, Cin, BNET_TC_ACT_NONE, 1, err_dev, stream);
}

// dw[Cout][3][3][Cin] = filter gradient of the same convolution: gy [N,H,W,Cout] and x [N,H,W,Cin] are read as 4-D TMA boxes of
// 64 pixels (the reduction), both MN-major; the pixel blocks are split over grid.z and the slice that arrives last at a tile
// converts the fp32 sums to bf16 (split-K fix-up).  `ws` (fp32 [Cout][9 Cin]) and `counters` (bnet_tc_conv3x3_wgrad_tiles ints)
// must be all zero on entry and are all zero again on exit.  splits <= 0: automatic.  Cin and Cout multiples of 64.
BNET_API int bnet_tc_conv3x3_wgrad(const void* gy, const void* x, void* dw, float* ws, int* counters, int N, int H, int W, int Cin,
                                   int Cout, int splits, int* err_dev, void* stream) {
  return run_conv_wgrad(gy, x, dw, ws, counters, N, H, W, Cin, Cout, splits, err_dev, stream);
}
BNET_API int bnet_tc_conv3x3_wgrad_tiles(int Cin, int Cout) { return wgrad_max_tiles(Cin, Cout); }
// the tiling of a 3x3 convolution (pure host function, like bnet_tc_plan): Cred / Cn as bnet_tc_conv3x3 (forward: Cin / Cout) or
// bnet_tc_conv3x3_dgrad (dgrad = 1: Cout / Cin) passes them to setup_conv; patch = {bw, bh, bn}, the pixels of one 128-row tile
BNET_API int bnet_tc_conv3x3_plan(int N, int H, int W, int Cred, int Cn, int dgrad, BnetTcPlan* plan, int patch[3]) {
  if (!plan || !patch) { g_err = "null plan"; return -1; }
  ConvProblem cp;
  uint16_t dummy[8] = {};
  int err_dummy = 0;
  if (const char* e = setup_conv(dummy, dummy, nullptr, dummy, N, H, W, Cred, Cn, BNET_TC_ACT_NONE, dgrad, &err_dummy, sm_count(), &cp)) {
    g_err = e;
    return -1;
  }
  *plan = cp.plan;
  patch[0] = cp.args.conv.bw;
  patch[1] = cp.args.conv.bh;
  patch[2] = cp.args.conv.bn;
  return 0;
}
// the tiling of a filter gradient (pure host function, like bnet_tc_plan): grid_x x grid_y tiles of 128 x bn, grid_z slices of
// the k_blocks 64-pixel blocks, ctas per slice
BNET_API int bnet_tc_conv3x3_wgrad_plan(int N, int H, int W, int Cin, int Cout, int splits, BnetTcPlan* plan) {
  if (!plan) { g_err = "null plan"; return -1; }
  WgradProblem wp;
  float ws_dummy = 0.f;
  int counters_dummy = 0, err_dummy = 0;
  if (const char* e = setup_conv_wgrad(&ws_dummy, &ws_dummy, &ws_dummy, &ws_dummy, &counters_dummy, N, H, W, Cin, Cout, splits,
                                       &err_dummy, sm_count(), &wp)) {
    g_err = e;
    return -1;
  }
  *plan = wp.plan;
  return 0;
}

// Host check of the shared-memory descriptors the wgmma linear kernel issues (csrc/cuda/tc_gemm.cu) against the CuTe
// definitions of the same bit fields (cute/arch/mma_sm90_desc.hpp, cute/atom/mma_traits_sm90_gmma.hpp, from CUTLASS
// headers installed alongside Python packages): the kernel packs them by hand so that it needs no CUTLASS at build time;
// this test is the cross-check, built only when the headers are around (tests/test_utils.py skips otherwise).
//
//   g++ -std=c++17 -I<cutlass>/include -Iinclude csrc/tests/tc_desc_test.cc -ldl -o build/tests/tc_desc_test
//   build/tests/tc_desc_test bagua_net_b200/lib/libnccl-net.so
#include <dlfcn.h>
#include <stdint.h>
#include <stdio.h>

#include <cute/tensor.hpp>
#include <cute/arch/mma_sm90_desc.hpp>
#include <cute/atom/mma_traits_sm90_gmma.hpp>

#include "bnet/bnet_tc.h"

int main(int argc, char** argv) {
  const char* path = argc > 1 ? argv[1] : "bagua_net_b200/lib/libnccl-net.so";
  void* h = dlopen(path, RTLD_NOW | RTLD_LOCAL);
  if (!h) { fprintf(stderr, "dlopen %s: %s\n", path, dlerror()); return 2; }
  auto smem_desc = reinterpret_cast<uint64_t (*)(uint32_t)>(dlsym(h, "bnet_tc_smem_desc"));
  auto plan = reinterpret_cast<int (*)(int, int, int, int, int, BnetTcPlan*)>(dlsym(h, "bnet_tc_plan"));
  auto smem_desc_mn = reinterpret_cast<uint64_t (*)(uint32_t)>(dlsym(h, "bnet_tc_smem_desc_mn"));
  if (!smem_desc || !plan || !smem_desc_mn) { fprintf(stderr, "missing bnet_tc_* symbols\n"); return 2; }
  int bad = 0;
  using namespace cute;
  using T = bfloat16_t;
  alignas(1024) static T buf[256 * 64];

  // ---- K-major: what make_gmma_desc<Major::K> builds for tile_to_shape(Layout_K_SW128_Atom<bf16>, (rows, 64)):
  //      128-byte swizzle, SBO = 8 rows * 128 B = 64 sixteen-byte units (the leading byte offset is unused by the hardware
  //      for swizzled K-major layouts and not compared)
  {
    auto t = make_tensor(make_smem_ptr(buf), tile_to_shape(GMMA::Layout_K_SW128_Atom<T>{}, Shape<_64, _64>{}));
    // (a descriptor describes one MMA's K = 16 slice of the tile)
    GmmaDescriptor want = GMMA::make_gmma_desc<GMMA::Major::K>(local_tile(t, Shape<_64, _16>{}, make_coord(0, 0)));
    for (uint32_t addr : {0u, 1024u, 16384u, 0x2A400u, 200u * 1024u}) {
      GmmaDescriptor got(smem_desc(addr));
      if (got.bitfield.layout_type_ != want.bitfield.layout_type_ || got.bitfield.stride_byte_offset_ != want.bitfield.stride_byte_offset_ ||
          got.bitfield.base_offset_ != 0 || got.bitfield.start_address_ != uint16_t(addr >> 4)) {
        printf("K-major smem desc @%x: got %016llx (layout %u sbo %u), CuTe layout %u sbo %u\n", addr, (unsigned long long)got.desc_,
               unsigned(got.bitfield.layout_type_), unsigned(got.bitfield.stride_byte_offset_), unsigned(want.bitfield.layout_type_),
               unsigned(want.bitfield.stride_byte_offset_));
        bad++;
      }
      // advancing K by 16 elements (32 bytes) inside the swizzle row only moves the start-address field
      GmmaDescriptor k1 = got;
      k1.bitfield.start_address_ = uint16_t((addr + 32) >> 4);
      if (got.desc_ + 2 != k1.desc_) { printf("smem desc K advance @%x\n", addr); bad++; }
    }
    if (int(t.layout()(0, 16)) * 2 != 32) { printf("K-major K slice offset: %d\n", int(t.layout()(0, 16)) * 2); bad++; }
  }

  // ---- MN-major operands (the backward GEMMs): the descriptor CuTe derives for the layout our TMA boxes produce — 64-element
  //      MN atoms 8 KiB apart, 8-row reduction groups 1 KiB apart, i.e. tile_to_shape(Layout_MN_SW128_Atom, (MN, 64), Step<_2,_1>)
  {
    auto check_mn = [&](auto shape, const char* name) {
      auto t = make_tensor(make_smem_ptr(buf), tile_to_shape(GMMA::Layout_MN_SW128_Atom<T>{}, shape, Step<_2, _1>{}));
      GmmaDescriptor want = GMMA::make_gmma_desc<GMMA::Major::MN>(local_tile(t, Shape<decltype(size<0>(shape)), _16>{}, make_coord(0, 0)));
      GmmaDescriptor got(smem_desc_mn(0x4000));
      if (got.bitfield.leading_byte_offset_ != want.bitfield.leading_byte_offset_ ||
          got.bitfield.stride_byte_offset_ != want.bitfield.stride_byte_offset_ || got.bitfield.layout_type_ != want.bitfield.layout_type_ ||
          got.bitfield.start_address_ != (0x4000 >> 4) || got.bitfield.base_offset_ != 0) {
        printf("MN-major smem desc (%s): got lbo %u sbo %u layout %u, CuTe lbo %u sbo %u layout %u\n", name,
               unsigned(got.bitfield.leading_byte_offset_), unsigned(got.bitfield.stride_byte_offset_), unsigned(got.bitfield.layout_type_),
               unsigned(want.bitfield.leading_byte_offset_), unsigned(want.bitfield.stride_byte_offset_), unsigned(want.bitfield.layout_type_));
        bad++;
      }
      // a K = 16 slice starts two 8-row groups (2048 B) further: layout(0, 16) in elements * 2 B
      if (int(t.layout()(0, 16)) * 2 != 2048) { printf("MN-major K slice offset (%s): %d\n", name, int(t.layout()(0, 16)) * 2); bad++; }
      if (int(t.layout()(64, 0)) * 2 != 8192 && size<0>(shape) > 64) { printf("MN-major atom offset (%s): %d\n", name, int(t.layout()(64, 0)) * 2); bad++; }
    };
    check_mn(Shape<_128, _64>{}, "128x64");
    check_mn(Shape<_256, _64>{}, "256x64");
  }

  // ---- tiling plans (no GPU here: the library plans for the 132 SMs of an H100 SXM)
  struct Case { int M, N, K, reduce, splits, swap, bn, gx, gy, gz; } cases[] = {
      {32, 4096, 25088, 0, 1, 1, 32, 1, 32, 1},     // VGG16 classifier fc1 at batch 32: weights fill the accumulator rows
      {64, 4096, 4096, 0, 1, 1, 64, 1, 32, 1},
      {256, 1000, 4096, 0, 1, 0, 128, 8, 2, 1},
      {4096, 4096, 4096, 1, 1, 0, 256, 16, 32, 1},     // 512 tiles of 128 x 256 >= 132 SMs
      {1024, 4096, 4096, 0, 1, 0, 128, 32, 8, 1},      // 128 tiles of 128 x 256 would leave SMs idle: stay at 128 x 128
      {32, 4096, 25088, 1, 4, 1, 32, 1, 32, 4},     // split-K on top of the cross-rank adds
      {8, 16, 64, 1, 8, 1, 32, 1, 1, 1},            // one K block: nothing to split
      {8192, 8192, 8192, 0, 1, 0, 256, 32, 64, 1},  // 2048 tiles on 132 SMs: persistent
  };
  for (const Case& c : cases) {
    BnetTcPlan p;
    if (plan(c.M, c.N, c.K, c.reduce, c.splits, &p) != 0 || p.swap != c.swap || p.bn != c.bn || p.grid_x != c.gx ||
        p.grid_y != c.gy || p.grid_z != c.gz || p.smem_bytes + 1024 > 232448 || p.k_per_split * p.grid_z < p.k_blocks ||
        p.k_per_split * (p.grid_z - 1) >= p.k_blocks || p.ctas < 1 || p.ctas > p.grid_x * p.grid_y ||
        p.ctas * p.grid_z > 132 + p.grid_z) {
      printf("plan %dx%dx%d: swap %d bn %d grid %d %d %d smem %d\n", c.M, c.N, c.K, p.swap, p.bn, p.grid_x, p.grid_y, p.grid_z,
             p.smem_bytes);
      bad++;
    }
  }
  BnetTcPlan p;
  if (plan(8192, 8192, 8192, 0, 1, &p) != 0 || p.ctas != 132) { printf("persistent plan: ctas %d\n", p.ctas); bad++; }
  if (plan(32, 64, 100, 0, 1, &p) == 0) { printf("K = 100 must be rejected (row pitch not a multiple of 16 bytes)\n"); bad++; }
  printf("tc_desc_test: %s\n", bad ? "FAILED" : "ok");
  return bad ? 1 : 0;
}

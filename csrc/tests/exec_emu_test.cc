// CPU emulation test of the transport executor's data-movement bodies (csrc/cuda/exec_body.cuh): the same
// process_range()/cta_share() the sm_90a kernels inline, compiled by g++ and run as an emulated cluster
// (every CTA, every thread, serially) over every op, odd sizes and unaligned offsets, against scalar references.
// Serial emulation is exact here: each destination element is touched by exactly one thread.
// (tests/test_gpu.py::test_executor_copy_reduce_cast runs the real kernels against PyTorch on an H100.)
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "cuda/exec_body.cuh"

using namespace bnet::cuda;

static int g_fail = 0;
#define CHECK(cond, ...)                                                   \
  do {                                                                     \
    if (!(cond)) {                                                         \
      if (g_fail < 20) { printf("FAIL %s:%d  %s  ", __FILE__, __LINE__, #cond); printf(__VA_ARGS__); printf("\n"); } \
      g_fail++;                                                            \
    }                                                                      \
  } while (0)

static unsigned g_seed = 99;
static unsigned urand() { g_seed = g_seed * 1664525u + 1013904223u; return g_seed >> 8; }
static float frand() { return (urand() & 0xffff) / 8192.0f - 4.0f; }

// run one job the way a cluster of `csize` CTAs with `nthreads` threads each does
static void run_job(uint32_t op, const char* src, char* dst, size_t nbytes, int csize, int nthreads, float scale) {
  for (int crank = 0; crank < csize; crank++) {
    size_t b0, b1;
    cta_share(op, nbytes, (uint32_t)crank, (uint32_t)csize, &b0, &b1);
    for (int tid = 0; tid < nthreads; tid++)
      process_range(op, src + b0, dst + dst_offset_for(op, b0), b1 - b0, tid, nthreads, scale);
  }
}

struct Buf {   // 64-byte aligned storage with guard bytes on both sides
  std::vector<unsigned char> raw;
  unsigned char* p;
  size_t n;
  Buf(size_t bytes, size_t misalign) : raw(bytes + 256 + misalign, 0xA5), n(bytes) {
    uintptr_t a = ((uintptr_t)raw.data() + 127) & ~(uintptr_t)63;
    p = (unsigned char*)a + misalign;
  }
  bool guards_ok() const {
    for (const unsigned char* q = raw.data(); q < p; q++) if (*q != 0xA5) return false;
    for (const unsigned char* q = p + n; q < raw.data() + raw.size(); q++) if (*q != 0xA5) return false;
    return true;
  }
};

static const int kClusters[] = {1, 2, 4};
static const int kThreadsEmu[] = {32, 96};

static void test_copy() {
  const size_t sizes[] = {1, 15, 16, 17, 255, 4096, 4099, 65536 + 13, 300001};
  const size_t offs[][2] = {{0, 0}, {1, 1}, {3, 7}, {16, 4}, {4, 8}, {2, 0}};
  for (size_t n : sizes)
    for (auto& o : offs)
      for (int cs : kClusters)
        for (int nt : kThreadsEmu) {
          Buf s(n, o[0]), d(n, o[1]);
          for (size_t i = 0; i < n; i++) s.p[i] = (unsigned char)urand();
          memset(d.p, 0, n);
          run_job(OP_COPY, (const char*)s.p, (char*)d.p, n, cs, nt, 1.f);
          CHECK(memcmp(s.p, d.p, n) == 0, "copy n=%zu so=%zu do=%zu cs=%d nt=%d", n, o[0], o[1], cs, nt);
          CHECK(d.guards_ok(), "copy wrote outside n=%zu so=%zu do=%zu", n, o[0], o[1]);
        }
}

template <typename S, typename D, typename Ref>
static void test_elementwise(const char* name, uint32_t op, size_t src_elem, size_t dst_elem, float scale, S make_src, D init_dst, Ref check) {
  // element counts around the vector / batch / share boundaries; byte offsets that keep element alignment
  const size_t counts[] = {8, 16, 24, 1000, 4096, 4104, 100003 / 8 * 8, (1u << 16) + 8};
  const size_t soffs[] = {0, 16, src_elem * 4 > 16 ? 16 : src_elem * 4};   // aligned, aligned, (possibly) vector-misaligned
  for (size_t cnt : counts)
    for (size_t so : soffs)
      for (int cs : kClusters)
        for (int nt : kThreadsEmu) {
          Buf s(cnt * src_elem, so), d(cnt * dst_elem, so == 0 ? 0 : so == 16 ? 32 : 8), d0(cnt * dst_elem, 0);
          make_src(s.p, cnt);
          init_dst(d.p, cnt);
          memcpy(d0.p, d.p, cnt * dst_elem);
          run_job(op, (const char*)s.p, (char*)d.p, cnt * src_elem, cs, nt, scale);
          size_t bad = check(s.p, d0.p, d.p, cnt);
          CHECK(bad == (size_t)-1, "%s cnt=%zu so=%zu cs=%d nt=%d first bad element %zu", name, cnt, so, cs, nt, bad);
          CHECK(d.guards_ok(), "%s wrote outside cnt=%zu so=%zu", name, cnt, so);
        }
}

static float bf(const unsigned char* p, size_t i) { __nv_bfloat16 v; memcpy(&v, p + 2 * i, 2); return __bfloat162float(v); }
static float f32(const unsigned char* p, size_t i) { float v; memcpy(&v, p + 4 * i, 4); return v; }
static void put_bf(unsigned char* p, size_t i, float f) { __nv_bfloat16 v = __float2bfloat16(f); memcpy(p + 2 * i, &v, 2); }
static void put_f32(unsigned char* p, size_t i, float f) { memcpy(p + 4 * i, &f, 4); }
static float fp8(unsigned char b, __nv_fp8_interpretation_t fmt) {
  __half_raw h = __nv_cvt_fp8_to_halfraw(b, fmt);
  __half hh;
  memcpy(&hh, &h, sizeof(hh));
  return __half2float(hh);
}

int main() {
  test_copy();
  auto src_f32 = [](unsigned char* p, size_t n) { for (size_t i = 0; i < n; i++) put_f32(p, i, frand()); };
  auto src_bf = [](unsigned char* p, size_t n) { for (size_t i = 0; i < n; i++) put_bf(p, i, frand()); };
  auto dst_f32 = [](unsigned char* p, size_t n) { for (size_t i = 0; i < n; i++) put_f32(p, i, frand()); };
  auto dst_bf = [](unsigned char* p, size_t n) { for (size_t i = 0; i < n; i++) put_bf(p, i, frand()); };
  auto dst_bytes = [](unsigned char* p, size_t n) { memset(p, 0x5a, n); };

  test_elementwise("red_add_f32", OP_RED_ADD_F32, 4, 4, 1.f, src_f32, dst_f32,
                   [](const unsigned char* s, const unsigned char* d0, const unsigned char* d, size_t n) {
                     for (size_t i = 0; i < n; i++) if (f32(d, i) != f32(d0, i) + f32(s, i)) return i;
                     return (size_t)-1;
                   });
  test_elementwise("red_add_bf16", OP_RED_ADD_BF16, 2, 2, 1.f, src_bf, dst_bf,
                   [](const unsigned char* s, const unsigned char* d0, const unsigned char* d, size_t n) {
                     for (size_t i = 0; i < n; i++) if (bf(d, i) != __bfloat162float(__float2bfloat16(bf(d0, i) + bf(s, i)))) return i;
                     return (size_t)-1;
                   });
  test_elementwise("cast_bf16_to_f32", OP_CAST_BF16_TO_F32, 2, 4, 1.f, src_bf, dst_f32,
                   [](const unsigned char* s, const unsigned char*, const unsigned char* d, size_t n) {
                     for (size_t i = 0; i < n; i++) if (f32(d, i) != bf(s, i)) return i;
                     return (size_t)-1;
                   });
  test_elementwise("acc_bf16_to_f32", OP_ACC_BF16_TO_F32, 2, 4, 1.f, src_bf, dst_f32,
                   [](const unsigned char* s, const unsigned char* d0, const unsigned char* d, size_t n) {
                     for (size_t i = 0; i < n; i++) if (f32(d, i) != f32(d0, i) + bf(s, i)) return i;
                     return (size_t)-1;
                   });
  test_elementwise("cast_f32_to_bf16", OP_CAST_F32_TO_BF16, 4, 2, 1.f, src_f32, dst_bf,
                   [](const unsigned char* s, const unsigned char*, const unsigned char* d, size_t n) {
                     for (size_t i = 0; i < n; i++) if (bf(d, i) != __bfloat162float(__float2bfloat16(f32(s, i)))) return i;
                     return (size_t)-1;
                   });
  const float scale = 16.f, inv = 1.f / 16.f;
  struct { const char* name; __nv_fp8_interpretation_t fmt; uint32_t from_bf16, from_f32, acc, to_f32; } fmts[] = {
      {"e4m3", __NV_E4M3, OP_CAST_BF16_TO_E4M3, OP_CAST_F32_TO_E4M3, OP_ACC_E4M3_TO_F32, OP_CAST_E4M3_TO_F32},
      {"e5m2", __NV_E5M2, OP_CAST_BF16_TO_E5M2, OP_CAST_F32_TO_E5M2, OP_ACC_E5M2_TO_F32, OP_CAST_E5M2_TO_F32}};
  for (auto& F : fmts) {
    const __nv_fp8_interpretation_t fmt = F.fmt;
    char nm[64];
    snprintf(nm, sizeof(nm), "cast_bf16_to_%s", F.name);
    test_elementwise(nm, F.from_bf16, 2, 1, scale, src_bf, dst_bytes,
                     [&](const unsigned char* s, const unsigned char*, const unsigned char* d, size_t n) {
                       for (size_t i = 0; i < n; i++)
                         if (d[i] != (unsigned char)__nv_cvt_float_to_fp8(bf(s, i) * scale, __NV_SATFINITE, fmt)) return i;
                       return (size_t)-1;
                     });
    snprintf(nm, sizeof(nm), "cast_f32_to_%s", F.name);
    test_elementwise(nm, F.from_f32, 4, 1, scale, src_f32, dst_bytes,
                     [&](const unsigned char* s, const unsigned char*, const unsigned char* d, size_t n) {
                       for (size_t i = 0; i < n; i++)
                         if (d[i] != (unsigned char)__nv_cvt_float_to_fp8(f32(s, i) * scale, __NV_SATFINITE, fmt)) return i;
                       return (size_t)-1;
                     });
    snprintf(nm, sizeof(nm), "acc_%s_to_f32", F.name);
    test_elementwise(nm, F.acc, 1, 4, inv,
                     [&](unsigned char* p, size_t n) {
                       for (size_t i = 0; i < n; i++) {          // any finite fp8 code (skip the NaN / Inf encodings)
                         unsigned char b = (unsigned char)urand();
                         float v = fp8(b, fmt);
                         p[i] = (v == v && fabsf(v) < 1e30f) ? b : (unsigned char)0x3c;
                       }
                     },
                     dst_f32,
                     [&](const unsigned char* s, const unsigned char* d0, const unsigned char* d, size_t n) {
                       for (size_t i = 0; i < n; i++) if (f32(d, i) != f32(d0, i) + fp8(s[i], fmt) * inv) return i;
                       return (size_t)-1;
                     });
    snprintf(nm, sizeof(nm), "cast_%s_to_f32", F.name);
    test_elementwise(nm, F.to_f32, 1, 4, inv,
                     [&](unsigned char* p, size_t n) {
                       for (size_t i = 0; i < n; i++) {
                         unsigned char b = (unsigned char)urand();
                         float v = fp8(b, fmt);
                         p[i] = (v == v && fabsf(v) < 1e30f) ? b : (unsigned char)0x3c;
                       }
                     },
                     dst_f32,
                     [&](const unsigned char* s, const unsigned char*, const unsigned char* d, size_t n) {
                       for (size_t i = 0; i < n; i++) if (f32(d, i) != fp8(s[i], fmt) * inv) return i;
                       return (size_t)-1;
                     });
  }
  printf("%s (%d failure%s)\n", g_fail ? "FAILED" : "executor body emulation tests passed", g_fail, g_fail == 1 ? "" : "s");
  return g_fail ? 1 : 0;
}

// CPU emulation test of the fused NHWC layer kernels: compiles the per-thread bodies of
// csrc/cuda/nn_body.cuh with g++ and walks an emulated grid (every block, every thread, serially), then
// compares with a straightforward scalar reference.  Checks the strided row walk, the tail handling of the
// unrolled load batches, the pool index coding and that every output element is written exactly as expected.
// (The same kernels are compared against PyTorch on a real H100 by tests/test_gpu.py::test_fused_nn.)
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "cuda/nn_body.cuh"

using namespace bnet::nn;

static int g_fail = 0;
#define CHECK(cond, ...)                                                   \
  do {                                                                     \
    if (!(cond)) {                                                         \
      if (g_fail < 20) { printf("FAIL %s:%d  %s  ", __FILE__, __LINE__, #cond); printf(__VA_ARGS__); printf("\n"); } \
      g_fail++;                                                            \
    }                                                                      \
  } while (0)

static unsigned g_seed = 12345;
static float frand() {   // uniform in [-2, 2), exactly representable in bf16 after rounding below
  g_seed = g_seed * 1664525u + 1013904223u;
  return ((g_seed >> 8) & 0xffff) / 16384.0f - 2.0f;
}

template <typename T> struct Conv;
template <> struct Conv<float> {
  static float to(float f) { return f; }
  static float from(float v) { return v; }
  static const char* name() { return "f32"; }
};
template <> struct Conv<__nv_bfloat16> {
  static __nv_bfloat16 to(float f) { return __float2bfloat16(f); }
  static float from(__nv_bfloat16 v) { return __bfloat162float(v); }
  static const char* name() { return "bf16"; }
};

template <typename T> static bool same(T a, T b) { return memcmp(&a, &b, sizeof(T)) == 0; }

template <typename T>
static void test_bias_relu(size_t rows, int C, int nblocks) {
  constexpr int V = Vec<T>::N;
  const int cvec = C / V;
  std::vector<T> z(rows * C), z0, bias(C);
  for (auto& v : z) v = Conv<T>::to(frand());
  for (auto& v : bias) v = Conv<T>::to(frand() * 0.5f);
  z0 = z;
  const size_t gthreads = (size_t)nblocks * 256;
  for (size_t t = 0; t < gthreads; t++) bias_relu_thread<T>(z.data(), bias.data(), rows * cvec, cvec, t, gthreads);
  for (size_t i = 0; i < rows * C; i++) {
    float e = fmaxf(Conv<T>::from(z0[i]) + Conv<T>::from(bias[i % C]), 0.f);
    CHECK(same(z[i], Conv<T>::to(e)), "%s bias_relu rows=%zu C=%d i=%zu", Conv<T>::name(), rows, C, i);
  }
}

template <typename T>
static void test_relu_bwd(size_t rows, int C, int nblocks) {
  constexpr int V = Vec<T>::N;
  const int cvec = C / V;
  const int threads = (256 / cvec) * cvec, rpb = threads / cvec;
  std::vector<T> gy(rows * C), y(rows * C), gz(rows * C);
  for (size_t i = 0; i < rows * C; i++) {
    gy[i] = Conv<T>::to(frand());
    float a = frand();
    y[i] = Conv<T>::to(a > 0.3f ? a : 0.f);     // post-ReLU activations: many exact zeros
  }
  memset((void*)gz.data(), 0x7f, gz.size() * sizeof(T));   // sentinel: every element must be overwritten
  std::vector<double> gb(C, 0.0);
  for (int b = 0; b < nblocks; b++)
    for (int t = 0; t < threads; t++) {
      float acc[V];
      for (int k = 0; k < V; k++) acc[k] = 0.f;
      relu_bwd_thread<T, 4>(gy.data(), y.data(), gz.data(), rows, cvec, rpb, t % cvec, t / cvec, (size_t)b, (size_t)nblocks, acc);
      for (int k = 0; k < V; k++) gb[(t % cvec) * V + k] += acc[k];
    }
  std::vector<double> ref(C, 0.0);
  for (size_t i = 0; i < rows * C; i++) {
    float e = Conv<T>::from(y[i]) > 0.f ? Conv<T>::from(gy[i]) : 0.f;
    CHECK(same(gz[i], Conv<T>::to(e)), "%s relu_bwd rows=%zu C=%d blocks=%d i=%zu", Conv<T>::name(), rows, C, nblocks, i);
    ref[i % C] += e;
  }
  for (int c = 0; c < C; c++)
    CHECK(fabs(gb[c] - ref[c]) <= 1e-3 * (1.0 + fabs(ref[c])), "%s relu_bwd bias grad c=%d %f vs %f", Conv<T>::name(), c, gb[c], ref[c]);
}

template <typename T>
static void test_pool(int N, int H, int W, int C, int nblocks) {
  constexpr int V = Vec<T>::N;
  const int cvec = C / V, Ho = H / 2, Wo = W / 2;
  const size_t in = (size_t)N * H * W * C, out = (size_t)N * Ho * Wo * C;
  std::vector<T> z(in), bias(C), p(out), gp(out), gz(in);
  std::vector<uint8_t> idx(out, 0xff);
  for (auto& v : z) v = Conv<T>::to(frand());
  for (auto& v : bias) v = Conv<T>::to(frand() * 0.5f);
  for (auto& v : gp) v = Conv<T>::to(frand());
  // ---- forward
  const size_t gthreads = (size_t)nblocks * 256;
  for (size_t t = 0; t < gthreads; t++)
    bias_relu_pool_fwd_thread<T>(z.data(), bias.data(), p.data(), idx.data(), N, H, W, cvec, t, gthreads);
  auto at = [&](int n, int h, int w, int c) { return (((size_t)n * H + h) * W + w) * C + c; };
  for (int n = 0; n < N; n++)
    for (int ho = 0; ho < Ho; ho++)
      for (int wo = 0; wo < Wo; wo++)
        for (int c = 0; c < C; c++) {
          float m = Conv<T>::from(z[at(n, 2 * ho, 2 * wo, c)]);
          int a = 0;
          for (int q = 1; q < 4; q++) {
            float v = Conv<T>::from(z[at(n, 2 * ho + q / 2, 2 * wo + q % 2, c)]);
            if (v > m) { m = v; a = q; }
          }
          m += Conv<T>::from(bias[c]);
          size_t o = (((size_t)n * Ho + ho) * Wo + wo) * C + c;
          CHECK(same(p[o], Conv<T>::to(fmaxf(m, 0.f))), "%s pool fwd value o=%zu", Conv<T>::name(), o);
          CHECK(idx[o] == (uint8_t)(a | (m > 0.f ? 4 : 0)), "%s pool fwd code o=%zu got %u", Conv<T>::name(), o, idx[o]);
        }
  // ---- backward through the codes
  const int threads = (256 / cvec) * cvec, rpb = threads / cvec;
  memset((void*)gz.data(), 0x7f, gz.size() * sizeof(T));
  std::vector<double> gb(C, 0.0), ref(C, 0.0);
  for (int b = 0; b < nblocks; b++)
    for (int t = 0; t < threads; t++) {
      float acc[V];
      for (int k = 0; k < V; k++) acc[k] = 0.f;
      pool_relu_bwd_thread<T, 4>(gp.data(), idx.data(), gz.data(), N, H, W, cvec, rpb, t % cvec, t / cvec, (size_t)b,
                                 (size_t)nblocks, acc);
      for (int k = 0; k < V; k++) gb[(t % cvec) * V + k] += acc[k];
    }
  for (int n = 0; n < N; n++)
    for (int ho = 0; ho < Ho; ho++)
      for (int wo = 0; wo < Wo; wo++)
        for (int c = 0; c < C; c++) {
          size_t o = (((size_t)n * Ho + ho) * Wo + wo) * C + c;
          float g = (idx[o] & 4) ? Conv<T>::from(gp[o]) : 0.f;
          ref[c] += g;
          for (int q = 0; q < 4; q++) {
            float e = ((idx[o] & 3) == q) ? g : 0.f;
            CHECK(same(gz[at(n, 2 * ho + q / 2, 2 * wo + q % 2, c)], Conv<T>::to(e)), "%s pool bwd N=%d H=%d W=%d C=%d o=%zu q=%d",
                  Conv<T>::name(), N, H, W, C, o, q);
          }
        }
  for (int c = 0; c < C; c++)
    CHECK(fabs(gb[c] - ref[c]) <= 1e-3 * (1.0 + fabs(ref[c])), "%s pool bwd bias grad c=%d %f vs %f", Conv<T>::name(), c, gb[c], ref[c]);
}

template <typename T>
static void test_bn(size_t rows, int C, int nblocks, bool relu, bool with_res) {
  constexpr int V = Vec<T>::N;
  const int cvec = C / V;
  const int threads = (256 / cvec) * cvec, rpb = threads / cvec;
  const float eps = 1e-5f;
  const bool bf = sizeof(T) == 2;
  std::vector<T> z(rows * C), res(rows * C), y(rows * C), gy(rows * C), gz(rows * C), gres(rows * C), gamma(C), beta(C);
  for (size_t i = 0; i < rows * C; i++) {
    z[i] = Conv<T>::to(frand() * (1.0f + (float)(i % C) / C) + 0.25f * (float)((i % C) % 5));   // channel-dependent mean / spread
    res[i] = Conv<T>::to(frand());
    gy[i] = Conv<T>::to(frand());
  }
  for (int c = 0; c < C; c++) {
    gamma[c] = Conv<T>::to(0.5f + 0.01f * (c % 37));
    beta[c] = Conv<T>::to(-0.3f + 0.02f * (c % 11));
  }
  // ---- statistics
  std::vector<double> st(2 * C, 0.0);
  for (int b = 0; b < nblocks; b++)
    for (int t = 0; t < threads; t++) {
      float acc[2 * V];
      for (int k = 0; k < 2 * V; k++) acc[k] = 0.f;
      bn_stats_thread<T, 4>(z.data(), rows, cvec, rpb, t % cvec, t / cvec, (size_t)b, (size_t)nblocks, acc);
      for (int k = 0; k < V; k++) {
        st[(t % cvec) * V + k] += acc[k];
        st[C + (t % cvec) * V + k] += acc[V + k];
      }
    }
  std::vector<double> rsum(C, 0.0), rsq(C, 0.0);
  for (size_t i = 0; i < rows * C; i++) {
    double v = Conv<T>::from(z[i]);
    rsum[i % C] += v;
    rsq[i % C] += v * v;
  }
  for (int c = 0; c < C; c++) {
    CHECK(fabs(st[c] - rsum[c]) <= 1e-3 * (1.0 + fabs(rsum[c])), "%s bn sum c=%d %f vs %f", Conv<T>::name(), c, st[c], rsum[c]);
    CHECK(fabs(st[C + c] - rsq[c]) <= 1e-3 * (1.0 + fabs(rsq[c])), "%s bn sumsq c=%d", Conv<T>::name(), c);
  }
  std::vector<float> stats(2 * C);
  for (int i = 0; i < 2 * C; i++) stats[i] = (float)st[i];
  const float inv_m = 1.0f / (float)rows;
  // ---- forward
  memset((void*)y.data(), 0x7f, y.size() * sizeof(T));
  for (int b = 0; b < nblocks; b++)
    for (int t = 0; t < threads; t++) {
      const int grp = t % cvec;
      float mean[V], invstd[V], var[V], scale[V], shift[V];
      bn_moments<V>(stats.data(), C, grp, inv_m, eps, mean, invstd, var);
      for (int k = 0; k < V; k++) {
        scale[k] = Conv<T>::from(gamma[grp * V + k]) * invstd[k];
        shift[k] = Conv<T>::from(beta[grp * V + k]) - mean[k] * scale[k];
      }
      bn_apply_thread<T, 4>(z.data(), with_res ? res.data() : nullptr, y.data(), rows, cvec, rpb, grp, t / cvec, (size_t)b,
                            (size_t)nblocks, scale, shift, relu);
    }
  std::vector<double> mean(C), invstd(C);
  for (int c = 0; c < C; c++) {
    mean[c] = rsum[c] / rows;
    double var = rsq[c] / rows - mean[c] * mean[c];
    invstd[c] = 1.0 / sqrt((var > 0 ? var : 0) + eps);
  }
  const double tol_y = bf ? 2e-2 : 2e-4;
  for (size_t i = 0; i < rows * C; i++) {
    const int c = (int)(i % C);
    double v = (Conv<T>::from(z[i]) - mean[c]) * invstd[c] * Conv<T>::from(gamma[c]) + Conv<T>::from(beta[c]);
    if (with_res) v += Conv<T>::from(res[i]);
    if (relu && v < 0) v = 0;
    CHECK(fabs(Conv<T>::from(y[i]) - v) <= tol_y * (1.0 + fabs(v)), "%s bn fwd rows=%zu C=%d i=%zu got %f want %f", Conv<T>::name(), rows, C,
          i, Conv<T>::from(y[i]), v);
  }
  // ---- backward
  std::vector<double> gs(2 * C, 0.0), r1(C, 0.0), r2(C, 0.0);
  for (int b = 0; b < nblocks; b++)
    for (int t = 0; t < threads; t++) {
      const int grp = t % cvec;
      float mn[V], is[V], var[V], acc[2 * V];
      bn_moments<V>(stats.data(), C, grp, inv_m, eps, mn, is, var);
      for (int k = 0; k < 2 * V; k++) acc[k] = 0.f;
      bn_bwd_reduce_thread<T, 2>(gy.data(), y.data(), z.data(), rows, cvec, rpb, grp, t / cvec, (size_t)b, (size_t)nblocks, mn, is, relu, acc);
      for (int k = 0; k < V; k++) {
        gs[grp * V + k] += acc[k];
        gs[C + grp * V + k] += acc[V + k];
      }
    }
  for (size_t i = 0; i < rows * C; i++) {
    const int c = (int)(i % C);
    double dy = (!relu || Conv<T>::from(y[i]) > 0.f) ? Conv<T>::from(gy[i]) : 0.0;
    r1[c] += dy;
    r2[c] += dy * (Conv<T>::from(z[i]) - mean[c]) * invstd[c];
  }
  for (int c = 0; c < C; c++) {
    CHECK(fabs(gs[c] - r1[c]) <= 2e-3 * (1.0 + fabs(r1[c])), "%s bn s1 c=%d %f vs %f", Conv<T>::name(), c, gs[c], r1[c]);
    CHECK(fabs(gs[C + c] - r2[c]) <= 2e-3 * (1.0 + fabs(r2[c])), "%s bn s2 c=%d %f vs %f", Conv<T>::name(), c, gs[C + c], r2[c]);
  }
  std::vector<float> gsum(2 * C);
  for (int i = 0; i < 2 * C; i++) gsum[i] = (float)gs[i];
  memset((void*)gz.data(), 0x7f, gz.size() * sizeof(T));
  memset((void*)gres.data(), 0x7f, gres.size() * sizeof(T));
  for (int b = 0; b < nblocks; b++)
    for (int t = 0; t < threads; t++) {
      const int grp = t % cvec;
      float mn[V], is[V], var[V], a[V], c1[V], c2[V];
      bn_moments<V>(stats.data(), C, grp, inv_m, eps, mn, is, var);
      for (int k = 0; k < V; k++) {
        a[k] = Conv<T>::from(gamma[grp * V + k]) * is[k];
        c1[k] = gsum[grp * V + k] * inv_m;
        c2[k] = gsum[C + grp * V + k] * inv_m;
      }
      bn_bwd_apply_thread<T, 2>(gy.data(), y.data(), z.data(), gz.data(), with_res ? gres.data() : nullptr, rows, cvec, rpb, grp,
                                t / cvec, (size_t)b, (size_t)nblocks, mn, is, a, c1, c2, relu);
    }
  const double tol_g = bf ? 2e-2 : 5e-4;
  for (size_t i = 0; i < rows * C; i++) {
    const int c = (int)(i % C);
    double dy = (!relu || Conv<T>::from(y[i]) > 0.f) ? Conv<T>::from(gy[i]) : 0.0;
    double xhat = (Conv<T>::from(z[i]) - mean[c]) * invstd[c];
    double want = Conv<T>::from(gamma[c]) * invstd[c] * (dy - r1[c] / rows - xhat * r2[c] / rows);
    CHECK(fabs(Conv<T>::from(gz[i]) - want) <= tol_g * (1.0 + fabs(want)), "%s bn bwd rows=%zu C=%d i=%zu got %f want %f", Conv<T>::name(),
          rows, C, i, Conv<T>::from(gz[i]), want);
    if (with_res) CHECK(same(gres[i], Conv<T>::to((float)dy)), "%s bn gres i=%zu", Conv<T>::name(), i);
  }
}

template <typename T>
static void run_all() {
  constexpr int V = Vec<T>::N;
  // rows chosen around the batch boundaries: fewer rows than one block step, exact multiples, ragged tails
  const int Cs[] = {V, 8 * V, 64 * V > 512 ? 512 : 64 * V};
  for (int C : Cs) {
    const int cvec = C / V, rpb = ((256 / cvec) * cvec) / cvec;
    const size_t row_cases[] = {1, (size_t)rpb - 1 > 0 ? (size_t)rpb - 1 : 1, (size_t)rpb, (size_t)rpb * 3 * 4, (size_t)rpb * 3 * 4 + 1,
                                (size_t)rpb * 3 * 9 + 5, 1000};
    for (size_t rows : row_cases) {
      if (rows * C > (1u << 21)) continue;
      test_bias_relu<T>(rows, C, 3);
      test_relu_bwd<T>(rows, C, 3);
      test_relu_bwd<T>(rows, C, 1);
    }
  }
  test_pool<T>(1, 2, 2, V, 1);
  test_pool<T>(2, 4, 6, 2 * V, 2);
  test_pool<T>(3, 8, 8, 8 * V, 3);
  test_pool<T>(2, 14, 14, 64, 5);
  test_pool<T>(1, 6, 10, 512, 2);
  // BatchNorm family: channel counts of a ResNet-50 (64 .. 2048), ragged row counts, with/without ReLU and residual
  const int bnC[] = {V, 64, 256, V * 256 > 2048 ? 2048 : V * 256};
  for (int C : bnC) {
    const int rpb = ((256 / (C / V)) * (C / V)) / (C / V);
    // (a handful of rows per channel makes the variance itself ill-conditioned: start at 33)
    const size_t rowsv[] = {33, (size_t)rpb * 5 + 33, 257, 1000};
    for (size_t rows : rowsv) {
      if (rows * C > (1u << 20)) continue;
      test_bn<T>(rows, C, 3, true, false);
      test_bn<T>(rows, C, 2, true, true);
      test_bn<T>(rows, C, 1, false, false);
    }
  }
}

int main() {
  run_all<float>();
  run_all<__nv_bfloat16>();
  printf("%s (%d failure%s)\n", g_fail ? "FAILED" : "nn kernel emulation tests passed", g_fail, g_fail == 1 ? "" : "s");
  return g_fail ? 1 : 0;
}

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
// equal bits, or both NaN (a NaN's payload is not part of the contract)
template <typename T> static bool same_or_nan(T a, T b) {
  const float fa = Conv<T>::from(a), fb = Conv<T>::from(b);
  return same(a, b) || (fa != fa && fb != fb);
}

// torch's rules: relu(x) = x <= 0 ? 0 : x (NaN stays NaN); threshold_backward(g, y) = y <= 0 ? 0 : g (a NaN y passes g)
static float relu_ref(float x) { return x <= 0.f ? 0.f : x; }
static bool passes_ref(float y) { return !(y <= 0.f); }

// with `specials`, every 5th element of a tensor is NaN, +Inf, -Inf or -0 instead (what a diverged run feeds a layer)
static float special(size_t i) {
  static const float v[4] = {NAN, INFINITY, -INFINITY, -0.0f};
  return v[(i / 5) % 4];
}
template <typename T> static void sprinkle(std::vector<T>& t, size_t phase) {
  for (size_t i = phase % 5; i < t.size(); i += 5) t[i] = Conv<T>::to(special(i + phase));
}
// sums that hold a NaN on both sides agree
static bool close_sum(double got, double want) {
  if (got != got || want != want) return got != got && want != want;
  if (isinf(got) || isinf(want)) return got == want;
  return fabs(got - want) <= 1e-3 * (1.0 + fabs(want));
}

template <typename T>
static void test_bias_relu(size_t rows, int C, int nblocks, bool specials = false) {
  constexpr int V = Vec<T>::N;
  const int cvec = C / V;
  std::vector<T> z(rows * C), z0, bias(C);
  for (auto& v : z) v = Conv<T>::to(frand());
  for (auto& v : bias) v = Conv<T>::to(frand() * 0.5f);
  if (specials) { sprinkle(z, 0); sprinkle(bias, 3); }
  z0 = z;
  const size_t gthreads = (size_t)nblocks * 256;
  for (size_t t = 0; t < gthreads; t++) bias_relu_thread<T>(z.data(), bias.data(), rows * cvec, cvec, t, gthreads);
  for (size_t i = 0; i < rows * C; i++) {
    float e = relu_ref(Conv<T>::from(z0[i]) + Conv<T>::from(bias[i % C]));
    CHECK(same_or_nan(z[i], Conv<T>::to(e)), "%s bias_relu rows=%zu C=%d i=%zu", Conv<T>::name(), rows, C, i);
  }
}

template <typename T>
static void test_relu_bwd(size_t rows, int C, int nblocks, bool specials = false) {
  constexpr int V = Vec<T>::N;
  const int cvec = C / V;
  const int threads = (256 / cvec) * cvec, rpb = threads / cvec;
  std::vector<T> gy(rows * C), y(rows * C), gz(rows * C);
  for (size_t i = 0; i < rows * C; i++) {
    gy[i] = Conv<T>::to(frand());
    float a = frand();
    y[i] = Conv<T>::to(a > 0.3f ? a : 0.f);     // post-ReLU activations: many exact zeros
  }
  if (specials) { sprinkle(y, 0); sprinkle(gy, 2); }
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
    float e = passes_ref(Conv<T>::from(y[i])) ? Conv<T>::from(gy[i]) : 0.f;
    CHECK(same_or_nan(gz[i], Conv<T>::to(e)), "%s relu_bwd rows=%zu C=%d blocks=%d i=%zu", Conv<T>::name(), rows, C, nblocks, i);
    ref[i % C] += e;
  }
  for (int c = 0; c < C; c++)
    CHECK(close_sum(gb[c], ref[c]), "%s relu_bwd bias grad c=%d %f vs %f", Conv<T>::name(), c, gb[c], ref[c]);
}

template <typename T>
static void test_pool(int N, int H, int W, int C, int nblocks, bool specials = false) {
  constexpr int V = Vec<T>::N;
  const int cvec = C / V, Ho = H / 2, Wo = W / 2;
  const size_t in = (size_t)N * H * W * C, out = (size_t)N * Ho * Wo * C;
  std::vector<T> z(in), bias(C), p(out), gp(out), gz(in);
  std::vector<uint8_t> idx(out, 0xff);
  for (auto& v : z) v = Conv<T>::to(frand());
  for (auto& v : bias) v = Conv<T>::to(frand() * 0.5f);
  for (auto& v : gp) v = Conv<T>::to(frand());
  if (specials) {
    sprinkle(z, 1);
    bias[0] = Conv<T>::to(NAN);
    if (C > 1) bias[1] = Conv<T>::to(INFINITY);
    if (C > 2) bias[2] = Conv<T>::to(-INFINITY);
    // exact ties inside windows (the first maximum wins) and windows with two NaNs (the last one wins)
    for (size_t i = 0; i + 3 * C < in; i += 7 * C + 1) z[i + C] = z[i];
    for (size_t i = 2; i + (size_t)W * C < in; i += 11 * C + 3) { z[i] = Conv<T>::to(NAN); z[i + (size_t)W * C] = Conv<T>::to(NAN); }
  }
  // ---- forward
  const size_t gthreads = (size_t)nblocks * 256;
  for (size_t t = 0; t < gthreads; t++)
    bias_relu_pool_fwd_thread<T>(z.data(), bias.data(), p.data(), idx.data(), N, H, W, cvec, t, gthreads);
  auto at = [&](int n, int h, int w, int c) { return (((size_t)n * H + h) * W + w) * C + c; };
  for (int n = 0; n < N; n++)
    for (int ho = 0; ho < Ho; ho++)
      for (int wo = 0; wo < Wo; wo++)
        for (int c = 0; c < C; c++) {
          // torch's max_pool2d: the first maximum wins a tie, a NaN wins over any number (the last NaN over an earlier one)
          const float b = Conv<T>::from(bias[c]);
          float m = Conv<T>::from(z[at(n, 2 * ho, 2 * wo, c)]) + b;
          int a = 0;
          for (int q = 1; q < 4; q++) {
            float v = Conv<T>::from(z[at(n, 2 * ho + q / 2, 2 * wo + q % 2, c)]) + b;
            if (v > m || v != v) { m = v; a = q; }
          }
          size_t o = (((size_t)n * Ho + ho) * Wo + wo) * C + c;
          CHECK(same_or_nan(p[o], Conv<T>::to(relu_ref(m))), "%s pool fwd value o=%zu", Conv<T>::name(), o);
          CHECK(idx[o] == (uint8_t)(a | (passes_ref(m) ? 4 : 0)), "%s pool fwd code o=%zu got %u want %u", Conv<T>::name(), o, idx[o],
                (unsigned)(a | (passes_ref(m) ? 4 : 0)));
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
            CHECK(same_or_nan(gz[at(n, 2 * ho + q / 2, 2 * wo + q % 2, c)], Conv<T>::to(e)), "%s pool bwd N=%d H=%d W=%d C=%d o=%zu q=%d",
                  Conv<T>::name(), N, H, W, C, o, q);
          }
        }
  for (int c = 0; c < C; c++)
    CHECK(close_sum(gb[c], ref[c]), "%s pool bwd bias grad c=%d %f vs %f", Conv<T>::name(), c, gb[c], ref[c]);
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
  // ---- statistics: sums of z - K and (z - K)^2, K = the channel's value in row 0
  std::vector<double> st(2 * C, 0.0);
  for (int b = 0; b < nblocks; b++)
    for (int t = 0; t < threads; t++) {
      float acc[2 * V], piv[V];
      for (int k = 0; k < 2 * V; k++) acc[k] = 0.f;
      bn_pivot<T>(z.data(), t % cvec, piv);
      bn_stats_thread<T, 4>(z.data(), rows, cvec, rpb, t % cvec, t / cvec, (size_t)b, (size_t)nblocks, piv, acc);
      for (int k = 0; k < V; k++) {
        st[(t % cvec) * V + k] += acc[k];
        st[C + (t % cvec) * V + k] += acc[V + k];
      }
    }
  std::vector<double> rsum(C, 0.0), rsq(C, 0.0), dsum(C, 0.0), dsq(C, 0.0);
  for (size_t i = 0; i < rows * C; i++) {
    double v = Conv<T>::from(z[i]), d = v - Conv<T>::from(z[i % C]);
    rsum[i % C] += v;
    rsq[i % C] += v * v;
    dsum[i % C] += d;
    dsq[i % C] += d * d;
  }
  for (int c = 0; c < C; c++) {
    CHECK(fabs(st[c] - dsum[c]) <= 1e-3 * (1.0 + fabs(dsum[c])), "%s bn sum c=%d %f vs %f", Conv<T>::name(), c, st[c], dsum[c]);
    CHECK(fabs(st[C + c] - dsq[c]) <= 1e-3 * (1.0 + fabs(dsq[c])), "%s bn sumsq c=%d", Conv<T>::name(), c);
  }
  std::vector<float> stats(2 * C);
  for (int i = 0; i < 2 * C; i++) stats[i] = (float)st[i];
  const float inv_m = 1.0f / (float)rows;
  // ---- forward
  memset((void*)y.data(), 0x7f, y.size() * sizeof(T));
  for (int b = 0; b < nblocks; b++)
    for (int t = 0; t < threads; t++) {
      const int grp = t % cvec;
      float piv[V], mean[V], invstd[V], var[V], scale[V], shift[V];
      bn_pivot<T>(z.data(), grp, piv);
      bn_moments<V>(stats.data(), piv, C, grp, inv_m, eps, mean, invstd, var);
      for (int k = 0; k < V; k++) {
        scale[k] = Conv<T>::from(gamma[grp * V + k]) * invstd[k];
        shift[k] = Conv<T>::from(beta[grp * V + k]);
      }
      bn_apply_thread<T, 4>(z.data(), with_res ? res.data() : nullptr, y.data(), rows, cvec, rpb, grp, t / cvec, (size_t)b,
                            (size_t)nblocks, mean, scale, shift, relu);
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
      float piv[V], mn[V], is[V], var[V], acc[2 * V];
      bn_pivot<T>(z.data(), grp, piv);
      bn_moments<V>(stats.data(), piv, C, grp, inv_m, eps, mn, is, var);
      for (int k = 0; k < 2 * V; k++) acc[k] = 0.f;
      bn_bwd_reduce_thread<T, 2>(gy.data(), y.data(), z.data(), rows, cvec, rpb, grp, t / cvec, (size_t)b, (size_t)nblocks, mn, is, relu, acc);
      for (int k = 0; k < V; k++) {
        gs[grp * V + k] += acc[k];
        gs[C + grp * V + k] += acc[V + k];
      }
    }
  for (size_t i = 0; i < rows * C; i++) {
    const int c = (int)(i % C);
    double dy = (!relu || passes_ref(Conv<T>::from(y[i]))) ? Conv<T>::from(gy[i]) : 0.0;
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
      float piv[V], mn[V], is[V], var[V], a[V], c1[V], c2[V];
      bn_pivot<T>(z.data(), grp, piv);
      bn_moments<V>(stats.data(), piv, C, grp, inv_m, eps, mn, is, var);
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
    double dy = (!relu || passes_ref(Conv<T>::from(y[i]))) ? Conv<T>::from(gy[i]) : 0.0;
    double xhat = (Conv<T>::from(z[i]) - mean[c]) * invstd[c];
    double want = Conv<T>::from(gamma[c]) * invstd[c] * (dy - r1[c] / rows - xhat * r2[c] / rows);
    CHECK(fabs(Conv<T>::from(gz[i]) - want) <= tol_g * (1.0 + fabs(want)), "%s bn bwd rows=%zu C=%d i=%zu got %f want %f", Conv<T>::name(),
          rows, C, i, Conv<T>::from(gz[i]), want);
    if (with_res) CHECK(same(gres[i], Conv<T>::to((float)dy)), "%s bn gres i=%zu", Conv<T>::name(), i);
  }
}

// BatchNorm apply / backward with ReLU on activations holding NaN and +-Inf: mean 0, scale 1, beta 0 make y = relu(z), and the
// backward passes dy wherever torch's threshold_backward would (y NaN included)
template <typename T>
static void test_bn_specials(size_t rows, int C) {
  constexpr int V = Vec<T>::N;
  const int cvec = C / V, threads = (256 / cvec) * cvec, rpb = threads / cvec;
  std::vector<T> z(rows * C), y(rows * C), gy(rows * C), gz(rows * C), gres(rows * C);
  for (size_t i = 0; i < rows * C; i++) { z[i] = Conv<T>::to(frand()); gy[i] = Conv<T>::to(frand()); }
  sprinkle(z, 0);
  float one[V], zero[V];
  for (int k = 0; k < V; k++) { one[k] = 1.f; zero[k] = 0.f; }
  memset((void*)y.data(), 0x7f, y.size() * sizeof(T));
  for (int t = 0; t < threads; t++)
    bn_apply_thread<T, 4>(z.data(), nullptr, y.data(), rows, cvec, rpb, t % cvec, t / cvec, 0, 1, zero, one, zero, true);
  for (size_t i = 0; i < rows * C; i++)
    CHECK(same_or_nan(y[i], Conv<T>::to(relu_ref(Conv<T>::from(z[i])))), "%s bn apply relu i=%zu", Conv<T>::name(), i);
  // mean 0, invstd 1, a 1, c1 = c2 = 0: gz = dy - z * 0, and gres = dy
  std::vector<double> s1(C, 0.0);
  for (int t = 0; t < threads; t++) {
    float acc[2 * V];
    for (int k = 0; k < 2 * V; k++) acc[k] = 0.f;
    bn_bwd_reduce_thread<T, 2>(gy.data(), y.data(), z.data(), rows, cvec, rpb, t % cvec, t / cvec, 0, 1, zero, one, true, acc);
    for (int k = 0; k < V; k++) s1[(t % cvec) * V + k] += acc[k];
    bn_bwd_apply_thread<T, 2>(gy.data(), y.data(), z.data(), gz.data(), gres.data(), rows, cvec, rpb, t % cvec, t / cvec, 0, 1, zero, one,
                              one, zero, zero, true);
  }
  std::vector<double> r1(C, 0.0);
  for (size_t i = 0; i < rows * C; i++) {
    const float dy = passes_ref(Conv<T>::from(y[i])) ? Conv<T>::from(gy[i]) : 0.f;
    r1[i % C] += dy;
    CHECK(same_or_nan(gres[i], Conv<T>::to(dy)), "%s bn bwd gres i=%zu", Conv<T>::name(), i);
    const float want = dy - Conv<T>::from(z[i]) * 0.f;     // xhat * c2: NaN where z is not finite
    CHECK(same_or_nan(gz[i], Conv<T>::to(want)), "%s bn bwd gz i=%zu", Conv<T>::name(), i);
  }
  for (int c = 0; c < C; c++) CHECK(close_sum(s1[c], r1[c]), "%s bn bwd s1 c=%d", Conv<T>::name(), c);
}

// bn_stats as the GPU adds it up, in the kernels' float order: each thread's walk, the block's rows of threads in ascending
// order (reduce_bias_grad), then the blocks' partial rows b = g (mod 8) per g and the 8 sums in order (sum_rows_kernel)
template <typename T>
static std::vector<float> emu_bn_stats(const std::vector<T>& z, size_t rows, int C, int nblocks) {
  constexpr int V = Vec<T>::N;
  const int cvec = C / V, threads = (256 / cvec) * cvec, rpb = threads / cvec;
  std::vector<float> part((size_t)nblocks * 2 * C, 0.f);
  std::vector<float> acc((size_t)threads * 2 * V);
  for (int b = 0; b < nblocks; b++) {
    for (int t = 0; t < threads; t++) {
      float* a = &acc[(size_t)t * 2 * V];
      float piv[V];
      for (int k = 0; k < 2 * V; k++) a[k] = 0.f;
      bn_pivot<T>(z.data(), t % cvec, piv);
      bn_stats_thread<T, 4>(z.data(), rows, cvec, rpb, t % cvec, t / cvec, (size_t)b, (size_t)nblocks, piv, a);
    }
    for (int g = 0; g < cvec; g++)
      for (int k = 0; k < 2 * V; k++) {
        float s = 0.f;
        for (int r = 0; r < rpb; r++) s += acc[(size_t)(r * cvec + g) * 2 * V + k];
        part[(size_t)b * 2 * C + (k < V ? 0 : C) + g * V + k % V] = s;
      }
  }
  std::vector<float> stats(2 * C);
  for (int c = 0; c < 2 * C; c++) {
    float sums[8];
    for (int g = 0; g < 8; g++) {
      sums[g] = 0.f;
      for (int b = g; b < nblocks; b += 8) sums[g] += part[(size_t)b * 2 * C + c];
    }
    float t = sums[0];
    for (int g = 1; g < 8; g++) t += sums[g];
    stats[c] = 0.f + t;
  }
  return stats;
}

// BatchNorm statistics of channels far from zero: channel c holds off[c] + sd * N(0, 1), and mean / std reaches 2^10.  The
// variance must stay within 2^-16 of a two-pass float64 variance of the same values, the mean within
// 2^-22 |mean| + 2^-20 std; a constant channel has variance 0 exactly.  Plain sums of z and z^2 lose (mean / std)^2 * 2^-24.
// bf16: channels made of three adjacent bf16 values around 2^e (mean / std near 2^7).
template <typename T>
static void test_bn_offset(size_t rows, int C, int nblocks) {
  constexpr int V = Vec<T>::N;
  const bool bf = sizeof(T) == 2;
  const double ratios[] = {0, 4, 16, 64, 256, 1024};
  const int nr = bf ? 1 : 6;
  std::vector<T> z(rows * C);
  std::vector<double> sd(C);
  unsigned s = 777u + (unsigned)C;
  auto gauss = [&]() {   // sum of 4 uniforms, scaled to unit variance
    double a = 0;
    for (int i = 0; i < 4; i++) { s = s * 1664525u + 1013904223u; a += ((s >> 8) & 0xffff) / 65536.0 - 0.5; }
    return a * sqrt(3.0);
  };
  for (int c = 0; c < C; c++) sd[c] = ldexp(1.0, (c % 7) - 3);
  for (size_t i = 0; i < rows * C; i++) {
    const int c = (int)(i % C);
    double v;
    if (c == C - 1) v = 3.0 * sd[c];                                       // a constant channel
    else if (bf) v = ldexp(1.0 + ((s = s * 1664525u + 1013904223u) >> 16) % 3 / 128.0, (c % 9) - 4);
    else v = ratios[c % nr] * sd[c] + sd[c] * gauss();
    z[i] = Conv<T>::to((float)v);
  }
  const std::vector<float> stats = emu_bn_stats<T>(z, rows, C, nblocks);
  const float inv_m = 1.0f / (float)rows;
  double worst = 0;
  for (int grp = 0; grp < C / V; grp++) {
    float piv[V], mean[V], invstd[V], var[V];
    bn_pivot<T>(z.data(), grp, piv);
    bn_moments<V>(stats.data(), piv, C, grp, inv_m, 1e-5f, mean, invstd, var);
    for (int k = 0; k < V; k++) {
      const int c = grp * V + k;
      double m = 0, v = 0;
      for (size_t r = 0; r < rows; r++) m += Conv<T>::from(z[r * C + c]);
      m /= rows;
      for (size_t r = 0; r < rows; r++) { const double d = Conv<T>::from(z[r * C + c]) - m; v += d * d; }
      v /= rows;
      const double bv = ldexp(v, -16), bm = ldexp(fabs(m), -22) + ldexp(sqrt(v), -20);
      CHECK(fabs(var[k] - v) <= bv, "%s bn offset var rows=%zu C=%d c=%d mean/std=%.0f: %.9g vs %.9g (rel %.2e)", Conv<T>::name(), rows, C, c,
            fabs(m) / sqrt(v), var[k], v, fabs(var[k] - v) / v);
      CHECK(fabs(mean[k] - m) <= bm, "%s bn offset mean rows=%zu C=%d c=%d: %.9g vs %.9g", Conv<T>::name(), rows, C, c, mean[k], m);
      if (v == 0) CHECK(var[k] == 0.f && (double)mean[k] == m, "%s bn constant channel c=%d: var %g mean %g", Conv<T>::name(), c, var[k], mean[k]);
      if (v > 0) worst = fmax(worst, fabs(var[k] - v) / bv);
    }
  }
  printf("  %s bn statistics of offset channels, rows=%zu C=%d blocks=%d: worst var error / 2^-16 var = %.3f\n", Conv<T>::name(), rows, C,
         nblocks, worst);
}

// an Inf or a NaN in a channel (in row 0, the pivot, or further down) makes its variance NaN, as in eager torch; the other
// channels keep their statistics
template <typename T>
static void test_bn_stats_nonfinite(size_t rows, int C, int nblocks) {
  constexpr int V = Vec<T>::N;
  std::vector<T> z(rows * C);
  for (auto& v : z) v = Conv<T>::to(frand());
  const float bad[3] = {INFINITY, -INFINITY, NAN};
  // channel 3j+q gets bad[q] in row 0 (j = 0) or in row 5 + j (j > 0)
  const int nbad = C < 9 ? C : 9;
  for (int c = 0; c < nbad; c++) z[(c < 3 ? 0 : (size_t)(5 + c / 3) % rows) * C + c] = Conv<T>::to(bad[c % 3]);
  const std::vector<float> stats = emu_bn_stats<T>(z, rows, C, nblocks);
  for (int grp = 0; grp < C / V; grp++) {
    float piv[V], mean[V], invstd[V], var[V];
    bn_pivot<T>(z.data(), grp, piv);
    bn_moments<V>(stats.data(), piv, C, grp, 1.0f / (float)rows, 1e-5f, mean, invstd, var);
    for (int k = 0; k < V; k++) {
      const int c = grp * V + k;
      if (c < nbad)
        CHECK(var[k] != var[k] && invstd[k] != invstd[k], "%s bn stats: channel %d holds %g, var %g invstd %g (want NaN)", Conv<T>::name(), c,
              bad[c % 3], var[k], invstd[k]);
      else
        CHECK(var[k] == var[k] && var[k] > 0.f && mean[k] == mean[k], "%s bn stats: finite channel %d has var %g mean %g", Conv<T>::name(), c,
              var[k], mean[k]);
    }
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

// NaN / +-Inf in the inputs: the layers follow eager torch (NaN propagates through ReLU and wins a pooling window)
template <typename T>
static void run_specials() {
  constexpr int V = Vec<T>::N;
  test_bias_relu<T>(257, 8 * V, 3, true);
  test_relu_bwd<T>(257, 8 * V, 3, true);
  test_pool<T>(2, 6, 10, 8 * V, 3, true);
  test_pool<T>(3, 8, 8, 64, 2, true);
  test_bn_specials<T>(100, 8 * V);
}

// the reduce kernels' grid (row_grid in nn_kernels.cu) with the planner's 132 SMs and 2 blocks per SM
static int bn_grid(size_t rows, int C, int V) {
  const int cvec = C / V, rpb = ((256 / cvec) * cvec) / cvec;
  const size_t want = (rows + 8 * (size_t)rpb - 1) / (8 * (size_t)rpb);
  return want < 264 ? (int)want : 264;
}

// BatchNorm statistics at ResNet-50 shapes with channels far from zero, and non-finite values through the statistics
template <typename T>
static void run_bn_statistics() {
  constexpr int V = Vec<T>::N;
  const size_t layer1 = 8 * 56 * 56, stem = 32 * 112 * 112;
  test_bn_offset<T>(layer1, 64, bn_grid(layer1, 64, V));
  test_bn_offset<T>(stem, 64, bn_grid(stem, 64, V));
  test_bn_offset<T>(2 * 7 * 7, 256 * V, bn_grid(2 * 7 * 7, 256 * V, V));
  test_bn_offset<T>(2, 8 * V, 1);
  test_bn_stats_nonfinite<T>(257, 8 * V, 3);
  test_bn_stats_nonfinite<T>(layer1, 64, bn_grid(layer1, 64, V));
}

int main() {
  run_all<float>();
  run_all<__nv_bfloat16>();
  run_specials<float>();
  run_specials<__nv_bfloat16>();
  run_bn_statistics<float>();
  run_bn_statistics<__nv_bfloat16>();
  printf("%s (%d failure%s)\n", g_fail ? "FAILED" : "nn kernel emulation tests passed", g_fail, g_fail == 1 ? "" : "s");
  return g_fail ? 1 : 0;
}

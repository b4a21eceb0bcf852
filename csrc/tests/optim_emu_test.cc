// CPU test of the fused AdamW update: compiles the per-element body of csrc/cuda/optim_body.cuh (what
// bnet_fused_adamw_kernel inlines) with g++ and compares it with a long-double AdamW fed the same fp32 inputs and
// the same fp32 hyper-parameters.
//
// Bound (u = 2^-24, F = 4 * 2^-149 for results in the subnormal range).  With M = b1|m| + (1-b1)|g|,
// V = b2 v + (1-b2) g^2, S = lr / (1 - b1^t), D the reference denominator and m1, p2 the reference results:
//   |m - m1| <= 4u M + F,   |v - v1| <= 6u V + F,
//   |p - p2| <= 3u|p| + 2u|p2| + S/D (5u M + 10u|m1|) + F
// (every operation rounds once; the hyper-parameters' own rounding is shared with the reference).
// Non-finite inputs must give the reference's pattern: NaN where it is NaN, the same infinity where it is infinite.
// The reference follows the operation order of torch's fused AdamW kernel (m = b1*m + (1-b1)*g).
// (The kernel itself is compared against float64 on an H100 by tests/test_fused_adamw.py.)
#include <math.h>
#include <stdio.h>

#include "cuda/optim_body.cuh"

using namespace bnet::optim;

static int g_fail = 0, g_checks = 0;
static double g_worst = 0.0;
#define CHECK(cond, ...)                                                   \
  do {                                                                     \
    g_checks++;                                                            \
    if (!(cond)) {                                                         \
      if (g_fail < 20) { printf("FAIL %s:%d  %s  ", __FILE__, __LINE__, #cond); printf(__VA_ARGS__); printf("\n"); } \
      g_fail++;                                                            \
    }                                                                      \
  } while (0)

static unsigned g_seed = 2024;
static float urand() {   // uniform in [0, 1)
  g_seed = g_seed * 1664525u + 1013904223u;
  return (g_seed >> 8) / 16777216.0f;
}
static float srand_(float scale) { return (2.0f * urand() - 1.0f) * scale; }

typedef long double LD;
static const LD kU = ldexpl(1.0L, -24), kF = 4 * ldexpl(1.0L, -149);

struct Hp { float lr, b1, b2, eps, wd, gscale, step; };

// one element: kernel body vs long double; `label` names the case in failures
static void check_one(const Hp& h, float g, float p, float m, float v, const char* label) {
  const float hp[kHpWords] = {h.lr, h.b1, h.b2, h.eps, h.wd, h.gscale, h.step, 0.f};
  const AdamWCoef c = adamw_coef(hp);
  float kp = p, km = m, kv = v;
  adamw_update(g, kp, km, kv, c);

  const LD t = (LD)h.step + 1, b1 = h.b1, b2 = h.b2, lr = h.lr;
  const LD gg = (LD)g * (LD)h.gscale;
  const LD p1 = (LD)p * (1 - lr * (LD)h.wd);
  const LD m1 = b1 * m + (1 - b1) * gg;
  const LD v1 = b2 * v + (1 - b2) * gg * gg;
  const LD S = lr / (1 - powl(b1, t));
  const LD D = sqrtl(v1) / sqrtl(1 - powl(b2, t)) + (LD)h.eps;
  const LD p2 = p1 - S * m1 / D;

  struct { const char* what; float got; LD want, bound; } r[3] = {
      {"m", km, m1, 4 * kU * (b1 * fabsl((LD)m) + (1 - b1) * fabsl(gg)) + kF},
      {"v", kv, v1, 6 * kU * (b2 * fabsl((LD)v) + (1 - b2) * gg * gg) + kF},
      {"p", kp, p2, 3 * kU * fabsl((LD)p) + 2 * kU * fabsl(p2) +
                        S / D * (5 * kU * (b1 * fabsl((LD)m) + (1 - b1) * fabsl(gg)) + 10 * kU * fabsl(m1)) + kF},
  };
  for (auto& e : r) {
    if (isnan(e.want) || isinf(e.want)) {
      const bool ok = isnan(e.want) ? isnan(e.got) : (LD)e.got == e.want;
      CHECK(ok, "%s: %s got %g want %Lg (g=%g p=%g m=%g v=%g step=%g)", label, e.what, e.got, e.want, g, p, m, v, h.step);
      continue;
    }
    const LD err = fabsl((LD)e.got - e.want);
    const bool ok = isfinite(e.got) && err <= e.bound;
    CHECK(ok, "%s: %s got %.9g want %.12Lg err %Lg bound %Lg (g=%g p=%g m=%g v=%g step=%g wd=%g)", label, e.what, e.got,
          e.want, err, e.bound, g, p, m, v, h.step, h.wd);
    if (ok && e.bound > 0) g_worst = fmax(g_worst, (double)(err / e.bound));
  }
}

int main() {
  const float steps[] = {0.f, 1.f, 9.f, 99999.f};   // words of the hp block: t = 1, 2, 10, 10^5
  const Hp bases[] = {
      {1e-3f, 0.9f, 0.999f, 1e-8f, 0.f, 1.f, 0},      // torch defaults, Adam (no decay)
      {1e-3f, 0.9f, 0.999f, 1e-8f, 1e-2f, 1.f, 0},    // torch's AdamW default decay
      {3e-2f, 0.8f, 0.95f, 1e-6f, 0.1f, 0.125f, 0},   // larger lr and decay, gradient averaged over 8 ranks
      {1e-1f, 0.f, 0.f, 1e-8f, 0.f, 0.5f, 0},         // beta = 0: m = g, v = g^2 (the staggered-CTA test's setting)
  };
  // gradient classes: ordinary, eps-dominated (sqrt(v) << eps), huge (|g|^2 still below FLT_MAX), zero
  const struct { const char* name; float gscale; } classes[] = {{"ordinary", 3.f}, {"tiny", 1e-12f}, {"huge", 1e18f}, {"zero", 0.f}};
  for (const float st : steps)
    for (Hp h : bases) {
      h.step = st;
      for (const auto& cl : classes)
        for (int i = 0; i < 2000; i++) {
          const float g = srand_(cl.gscale);
          const float p = srand_(2.f);
          // state of the same magnitude as the gradients (half the time), or left over from larger ones
          const float ms = (i & 1) ? cl.gscale : 1.f;
          const float m = srand_(ms);
          const float v = urand() * ms * ms;
          check_one(h, g, p, m, v, cl.name);
        }
    }
  // non-finite values in g, m and v (p, m, v finite elsewhere)
  const float specials[] = {NAN, INFINITY, -INFINITY};
  for (const float st : steps)
    for (Hp h : bases) {
      h.step = st;
      for (const float s : specials) {
        check_one(h, s, 0.5f, 0.01f, 1e-4f, "g special");
        check_one(h, 0.3f, 0.5f, s, 1e-4f, "m special");
        check_one(h, 0.3f, 0.5f, 0.01f, s, "v special");
        check_one(h, s, 0.5f, s, s, "all special");
      }
    }
  // a NaN gradient poisons its own element only: the neighbours of the emulated vector are untouched by it
  {
    const float hp[kHpWords] = {1e-3f, 0.9f, 0.999f, 1e-8f, 1e-2f, 1.f, 0.f, 0.f};
    const AdamWCoef c = adamw_coef(hp);
    float g[8] = {0.1f, NAN, -0.2f, INFINITY, 0.3f, -INFINITY, 0.f, 1.f}, p[8], m[8], v[8];
    for (int k = 0; k < 8; k++) { p[k] = 0.5f; m[k] = 0.f; v[k] = 0.f; }
    for (int k = 0; k < 8; k++) adamw_update(g[k], p[k], m[k], v[k], c);
    for (int k = 0; k < 8; k++) {
      const bool special = k == 1 || k == 3 || k == 5;
      CHECK(isnan(p[k]) == special, "element %d: p=%g", k, p[k]);
      CHECK(isnan(m[k]) == (k == 1) && isnan(v[k]) == (k == 1), "element %d: m=%g v=%g", k, m[k], v[k]);
    }
  }
  printf("optim_emu_test: %d checks, %d failures, worst error/bound %.3f\n", g_checks, g_fail, g_worst);
  if (g_fail) return 1;
  printf("optim_emu_test: ok\n");
  return 0;
}

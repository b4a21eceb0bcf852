// CPU test of the fused optimizer updates: compiles the per-element bodies of csrc/cuda/optim_body.cuh (what
// bnet_fused_adamw_kernel and bnet_fused_sgd_kernel inline) with g++ and compares them with a long-double AdamW and SGD
// fed the same fp32 inputs and the same fp32 hyper-parameters.  The SGD part and its bound are further down, and so is
// the LARS trust ratio (lars_trust / lars_scalars) and the EMA gate and lerp (ema_gate / ema_lerp).
//
// AdamW:
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

static void adamw_checks() {
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
}

// ------------------------------------------------------------------ SGD
// One element through several steps: the kernel body (sgd_update, fed g, or fl(scratch * coef) on the clipped path)
// and a long-double torch.optim.SGD fed the same fp32 inputs and hyper-parameters, with G = g * coef * gscale:
//   d = wd p + G,   b' = mu b + d,   p' = p - lr b'
// with torch's treatment of zero hyper-parameters: d = G when wd = 0 (p is not read), b' = d when mu = 0 (no buffer).
// The kernel rounds g*gscale, the fmaf for d, the fmaf for b' and the one for p' (and scratch*coef before them on the
// clipped path).  To first order, with the bounds B of the step before carried forward:
//   B_d  = wd B_p + u(wd|p| + k|G|) + F             (k = 2, or 3 on the clipped path)
//   B_b' = mu B_b + B_d + u(mu|b| + |d|) + F
//   B_p' = B_p + lr B_b' + u(|p| + lr|b'|) + F
struct SgdHp { float lr, mu, wd, gs; };

struct SgdElem {
  float p, b;          // kernel state
  LD rp, rb;           // reference state
  LD Bp, Bb;           // bounds of |p - rp|, |b - rb|
};

static SgdElem sgd_elem(float p, float b) { return SgdElem{p, b, (LD)p, (LD)b, 0, 0}; }

static double s_worst = 0.0;

static void sgd_check(const char* what, float got, LD want, LD bound, const char* label, const SgdHp& h, float g) {
  if (isnan(want) || isinf(want)) {
    const bool ok = isnan(want) ? isnan(got) : (LD)got == want;
    CHECK(ok, "sgd %s: %s got %g want %Lg (g=%g lr=%g mu=%g wd=%g gs=%g)", label, what, got, want, g, h.lr, h.mu, h.wd, h.gs);
    return;
  }
  const LD err = fabsl((LD)got - want);
  // after a non-finite step the carried bound is no longer finite; a finite reference value then needs a finite result
  const bool ok = isfinite(got) && (!isfinite(bound) || err <= bound);
  CHECK(ok, "sgd %s: %s got %.9g want %.12Lg err %Lg bound %Lg (g=%g lr=%g mu=%g wd=%g gs=%g)", label, what, got, want, err,
        bound, g, h.lr, h.mu, h.wd, h.gs);
  if (ok && isfinite(bound) && bound > 0) s_worst = fmax(s_worst, (double)(err / bound));
}

// one step of element `e`; coef < 0: the one-kernel path, else the clipped path with that coefficient
static void sgd_step(SgdElem& e, const SgdHp& h, float g, float coef, const char* label) {
  const bool clipped = coef >= 0.0f;
  sgd_update(clipped ? g * coef : g, e.p, e.b, h.lr, h.mu, h.wd, h.gs);

  const LD lr = h.lr, mu = h.mu, wd = h.wd;
  const LD G = (LD)g * (clipped ? (LD)coef : 1.0L) * (LD)h.gs;
  const LD d = h.wd == 0.0f ? G : wd * e.rp + G;
  const LD b1 = h.mu == 0.0f ? d : mu * e.rb + d;
  const LD p1 = e.rp - lr * b1;
  const LD Bd = wd * e.Bp + kU * (wd * fabsl(e.rp) + (clipped ? 3 : 2) * fabsl(G)) + kF;
  const LD Bb = mu * e.Bb + Bd + kU * (mu * fabsl(e.rb) + fabsl(d)) + kF;
  const LD Bp = e.Bp + lr * Bb + kU * (fabsl(e.rp) + lr * fabsl(b1)) + kF;
  e.rp = p1, e.rb = b1, e.Bp = Bp, e.Bb = Bb;
  sgd_check("p", e.p, e.rp, e.Bp, label, h, g);
  sgd_check("buf", e.b, e.rb, e.Bb, label, h, g);
}

static void sgd_checks() {
  const SgdHp bases[] = {
      {0.1f, 0.9f, 1e-2f, 1.f},          // momentum and weight decay
      {0.05f, 0.f, 0.f, 0.5f},           // plain SGD (no buffer in torch), gradient averaged over 2 ranks
      {0.1f, 0.9f, 0.f, 1.f / 3},        // a gradient scale that is not a power of two (3 ranks)
      {0.f, 0.9f, 1e-2f, 1.f},           // lr = 0: the parameters stay, the buffer still moves
  };
  const float coefs[] = {-1.f, 0.3f, 1e-3f, 1.f, 0.f};     // the one-kernel path, then clipped with these coefficients
  // gradient classes: ordinary, tiny (subnormal products), huge, zero
  const struct { const char* name; float scale; } classes[] = {{"ordinary", 3.f}, {"tiny", 1e-36f}, {"huge", 1e30f}, {"zero", 0.f}};
  const float lr_sched[] = {1.f, 1.f, 0.3f, 0.3f, 0.1f};   // the learning rate changes between steps
  for (const SgdHp& h0 : bases)
    for (const float coef : coefs)
      for (const auto& cl : classes)
        for (int i = 0; i < 400; i++) {
          // state of the gradients' magnitude (half the time), or left over from larger ones; 5 steps
          const float ss = (i & 1) ? cl.scale : 1.f;
          SgdElem e = sgd_elem(srand_(2.f), (i & 2) ? srand_(ss) : 0.f);
          for (const float f : lr_sched) {
            SgdHp h = h0;
            h.lr = h0.lr * f;
            sgd_step(e, h, srand_(cl.scale), coef, cl.name);
          }
        }
  // NaN and +-Inf in g and in the buffer, one step from finite p
  const float specials[] = {NAN, INFINITY, -INFINITY};
  for (const SgdHp& h : bases)
    for (const float coef : coefs)
      for (const float s : specials) {
        SgdElem a = sgd_elem(0.5f, 0.01f), b = sgd_elem(0.5f, s), c = sgd_elem(0.5f, s);
        sgd_step(a, h, s, coef, "g special");
        sgd_step(b, h, 0.3f, coef, "buf special");
        sgd_step(c, h, s, coef, "all special");
      }
  // momentum 0 after an infinite gradient: torch steps with d_p alone, so the element stays at its infinity (or NaN)
  // and the next finite gradients do not turn it into NaN
  const float decays[] = {0.f, 1e-2f};
  for (const float wd : decays)
    for (const float s : specials) {
      const SgdHp h = {0.1f, 0.f, wd, 1.f};
      SgdElem e = sgd_elem(0.5f, 0.f), f = sgd_elem(0.5f, 0.f);
      sgd_step(e, h, s, -1.f, "mu=0 sequence");
      sgd_step(f, h, 0.3f, -1.f, "mu=0 sequence");
      for (int k = 0; k < 2; k++) {
        sgd_step(e, h, 0.3f, -1.f, "mu=0 sequence");
        sgd_step(f, h, 0.3f, -1.f, "mu=0 sequence");
      }
      if (wd == 0.f) {
        CHECK(isnan(s) ? isnan(e.p) : e.p == -s, "mu=0: p=%g after g=%g", e.p, s);
        CHECK(isfinite(e.b) && e.b == 0.3f, "mu=0: buf=%g (d_p of the last step)", e.b);
      }
      CHECK(isfinite(f.p), "mu=0: neighbour p=%g", f.p);
    }
}

// ---------------------------------------------------------------------------------------------------------- LARS
// lars_trust against long double on the same fp32 inputs: t = eta*wn / ((gn + wd*wn) + eps) takes four roundings
// (product, fma, add, divide) of non-negative terms, so |t - T| <= 4.5u T (+ F).  The special cases follow Apex's
// LARC: t = 1 when a norm is exactly 0, NaN from a NaN norm, 0 from an infinite gradient norm.  lars_scalars must give
// {t, gs*t, wd*t}, or {1, gs, 0} for excluded tensors and zero norms.
static double l_worst = 0.0;

static LD lars_ref(float eta, float eps, float wd, float wn, float gn) {
  return (LD)eta * wn / ((LD)gn + (LD)wd * wn + (LD)eps);
}

static void lars_checks() {
  const float etas[] = {1e-3f, 0.02f, 1.f};
  const float epss[] = {0.f, 1e-8f, 1e-3f};
  const float wds[] = {0.f, 5e-5f, 1e-4f, 0.1f};
  for (const float eta : etas)
    for (const float eps : epss)
      for (const float wd : wds)
        for (int i = 0; i < 4000; i++) {
          // norms from 2^-60 to 2^40: tiny and huge gradients, layers of any size
          const float wn = ldexpf(0.5f + urand(), (int)(urand() * 100.f) - 60);
          const float gn = ldexpf(0.5f + urand(), (int)(urand() * 100.f) - 60);
          const float t = lars_trust(eta, eps, wd, wn, gn);
          const LD T = lars_ref(eta, eps, wd, wn, gn);
          const LD bound = 4.5L * kU * fabsl(T) + kF;
          const LD err = fabsl((LD)t - T);
          CHECK(isfinite(t) && err <= bound, "lars_trust(%g, %g, %g, %g, %g) = %.9g, reference %.12Lg", eta, eps, wd, wn, gn, t, T);
          if ((double)(err / bound) > l_worst) l_worst = (double)(err / bound);
          const float gs = 0.125f * (0.5f + urand());
          const LarsScalars s = lars_scalars(eta, eps, wd, gs, wn, gn, false);
          CHECK(s.t == t && s.gscale == gs * t && s.wd == wd * t, "lars_scalars != {t, gs*t, wd*t}");
          const LarsScalars x = lars_scalars(eta, eps, wd, gs, wn, gn, true);
          CHECK(x.t == 1.f && x.gscale == gs && x.wd == 0.f, "excluded tensor: {%g, %g, %g}", x.t, x.gscale, x.wd);
        }
  // the special cases of Apex's LARC (clip=False)
  const float eta = 1e-3f, eps = 1e-8f, wd = 1e-4f;
  CHECK(lars_trust(eta, eps, wd, 0.f, 3.f) == 1.f, "wn == 0 -> 1");
  CHECK(lars_trust(eta, eps, wd, 3.f, 0.f) == 1.f, "gn == 0 -> 1");
  CHECK(lars_trust(eta, eps, wd, 0.f, 0.f) == 1.f, "both 0 -> 1");
  CHECK(lars_trust(eta, eps, wd, -0.f, 3.f) == 1.f, "wn == -0 -> 1");
  CHECK(isnan(lars_trust(eta, eps, wd, NAN, 3.f)), "NaN wn -> NaN");
  CHECK(isnan(lars_trust(eta, eps, wd, 3.f, NAN)), "NaN gn -> NaN");
  CHECK(isnan(lars_trust(eta, eps, wd, NAN, 0.f)) == false && lars_trust(eta, eps, wd, NAN, 0.f) == 1.f,
        "gn == 0 wins over a NaN wn, as Apex's 'and'");
  CHECK(lars_trust(eta, eps, wd, 3.f, INFINITY) == 0.f, "gn = inf -> 0");
  CHECK(isnan(lars_trust(eta, eps, wd, INFINITY, 3.f)), "wn = inf with wd > 0 -> inf / inf = NaN");
  CHECK(isnan(lars_trust(eta, eps, 0.f, INFINITY, 3.f)), "wn = inf with wd = 0 -> NaN (inf * 0 in the denominator, as Apex)");
  CHECK(lars_trust(eta, 0.f, 0.f, 2.f, 4.f) == eta * 0.5f, "eps = wd = 0: eta * wn / gn");
  const LarsScalars z = lars_scalars(eta, eps, wd, 0.25f, 3.f, 0.f, false);
  CHECK(z.t == 1.f && z.gscale == 0.25f && z.wd == 0.f, "zero gradient norm: no weight decay, as in Apex");
  const LarsScalars zw = lars_scalars(eta, eps, wd, 0.25f, 0.f, 2.f, false);
  CHECK(zw.t == 1.f && zw.gscale == 0.25f && zw.wd == 0.f, "zero weight norm: {1, gs, 0}");
  const LarsScalars n = lars_scalars(eta, eps, wd, 0.25f, 3.f, NAN, false);
  CHECK(isnan(n.t) && isnan(n.gscale) && isnan(n.wd), "NaN gradient norm poisons the tensor");
  const LarsScalars f = lars_scalars(eta, eps, wd, 0.25f, 3.f, INFINITY, false);
  CHECK(f.t == 0.f && f.gscale == 0.f && f.wd == 0.f, "infinite gradient norm: t = 0");
  const LarsScalars e = lars_scalars(eta, eps, wd, NAN, 3.f, 2.f, true);
  CHECK(e.t == 1.f && isnan(e.gscale) && e.wd == 0.f, "excluded tensor keeps a NaN clip coefficient in its scale");
}

// ---------------------------------------------------------------------------------------------------------- EMA
// ema_gate against integer arithmetic: step s + 1 updates when (s + 1) % every == 0, and the update is a copy when
// n_averaged == 0, for counters up to 2^24.  ema_lerp against torch.lerp's two branches in long double on the same fp32
// inputs: the difference and the fma round once each, so to first order |r - R| <= u(|R| + min(w, 1 - w)|m - e|) (+ F,
// and a factor 1 + 2^-13 for the second-order term); weight 0 gives
// the EMA and weight 1 the master exactly; NaN and +-Inf give what the same formula gives in IEEE arithmetic.
static double e_worst = 0.0;

static LD lerp_ref(float e, float m, float w) {
  const LD d = (LD)m - (LD)e;
  return fabsf(w) < 0.5f ? (LD)e + (LD)w * d : (LD)m - d * (1.0L - (LD)w);
}

static void ema_checks() {
  const unsigned everys[] = {1u, 2u, 3u, 7u, 32u, 1000u, 1u << 12, (1u << 23) + 1u, 1u << 23, 1u << 24};
  const unsigned steps[] = {0u, 1u, 2u, 6u, 30u, 31u, 32u, 999u, 4095u, 4096u, (1u << 23) - 1u, 1u << 23,
                            (1u << 24) - 2u, (1u << 24) - 1u};
  const float counts[] = {0.f, 1.f, 5.f, 16777216.f};
  for (const unsigned ev : everys)
    for (const unsigned s : steps)
      for (const float n : counts) {
        const EmaGate g = ema_gate((float)s, (float)ev, n);
        const bool due = (s + 1u) % ev == 0u;
        CHECK(g.update == due && g.copy == (due && n == 0.f), "ema_gate(step=%u, every=%u, n=%g) = {%d, %d}", s, ev, n,
              g.update, g.copy);
      }
  // a run of steps from 0, counting as bnet_ema_advance_kernel does
  const unsigned runs[] = {1u, 3u, 32u};
  for (const unsigned ev : runs) {
    float step = 0.f, n = 0.f;
    unsigned updates = 0, copies = 0;
    for (unsigned s = 1; s <= 1000; s++) {
      const EmaGate g = ema_gate(step, (float)ev, n);
      updates += g.update, copies += g.copy;
      if (g.update) n += 1.f;
      step += 1.f;
    }
    CHECK(updates == 1000 / ev && copies == 1 && n == (float)(1000 / ev) && step == 1000.f, "every=%u: %u updates, %u copies",
          ev, updates, copies);
  }
  const float weights[] = {0.f, 1.f, 2e-5f, 3.0517578e-4f, 1e-3f, 0.1f, 0.4999999f, 0.5f, 0.5000001f, 0.75f, 0.999f};
  for (const float w : weights)
    for (int i = 0; i < 20000; i++) {
      // EMA and master close to each other (the usual case), far apart, and of different magnitudes
      const float scale = ldexpf(1.f, (int)(urand() * 40.f) - 20);
      const float e = srand_(scale);
      const float m = (i & 1) ? e + srand_(scale * 1e-3f) : srand_(scale * ((i & 2) ? 1.f : 1e4f));
      const float r = ema_lerp(e, m, w);
      if (w == 0.f) { CHECK(r == e, "weight 0: %g, not the EMA %g", r, e); continue; }
      if (w == 1.f) { CHECK(r == m, "weight 1: %g, not the master %g", r, m); continue; }
      const LD R = lerp_ref(e, m, w);
      const LD bound = (1 + ldexpl(1.0L, -13)) * kU * (fabsl(R) + fminl((LD)w, 1.0L - (LD)w) * fabsl((LD)m - (LD)e)) + kF;
      const LD err = fabsl((LD)r - R);
      CHECK(isfinite(r) && err <= bound, "ema_lerp(%g, %g, %g) = %.9g, reference %.12Lg", e, m, w, r, R);
      if (bound > 0 && (double)(err / bound) > e_worst) e_worst = (double)(err / bound);
    }
  // NaN and +-Inf in either operand, in both branches
  const float specials[] = {NAN, INFINITY, -INFINITY, 0.5f};
  const float sweights[] = {0.f, 1e-3f, 0.75f, 1.f};
  for (const float w : sweights)
    for (const float e : specials)
      for (const float m : specials) {
        const float r = ema_lerp(e, m, w);
        const LD R = lerp_ref(e, m, w);
        CHECK(isnan(R) ? isnan(r) : (LD)r == R, "ema_lerp(%g, %g, %g) = %g, reference %Lg", e, m, w, r, R);
      }
  CHECK(isnan(ema_lerp(INFINITY, 1.f, 1e-3f)), "EMA +inf, finite master, small weight: inf - inf = NaN, as torch.lerp");
  CHECK(ema_lerp(1.f, INFINITY, 1e-3f) == INFINITY, "an infinite master makes the EMA infinite below weight 0.5");
  CHECK(isnan(ema_lerp(1.f, INFINITY, 0.75f)), "... and NaN above it (inf - inf * (1 - w)), as torch.lerp");
}

int main() {
  ema_checks();
  const int ema = g_checks;
  printf("optim_emu_test: ema %d checks, worst error/bound %.3f\n", ema, e_worst);
  lars_checks();
  const int lars = g_checks - ema;
  printf("optim_emu_test: lars %d checks, worst error/bound %.3f\n", lars, l_worst);
  adamw_checks();
  const int adamw = g_checks - lars - ema;
  printf("optim_emu_test: adamw %d checks, worst error/bound %.3f\n", adamw, g_worst);
  sgd_checks();
  printf("optim_emu_test: sgd %d checks, worst error/bound %.3f\n", g_checks - adamw - lars - ema, s_worst);
  printf("optim_emu_test: %d checks, %d failures\n", g_checks, g_fail);
  if (g_fail) return 1;
  printf("optim_emu_test: ok\n");
  return 0;
}

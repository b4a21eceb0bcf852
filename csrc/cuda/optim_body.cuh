// Per-element arithmetic of the fused optimizer kernels (csrc/cuda/coll.cu): sgd_update for
// bnet_fused_sgd_kernel and adamw_update for bnet_fused_adamw_kernel, clip_coef for the clipped step, lars_trust /
// lars_scalars for the LARS step, ema_gate / ema_lerp for the EMA of the master weights, and group_seg_find /
// group_seg_advance, the parameter-group lookup of the grouped SGD and AdamW kernels.
//
// The updates are written here as plain __host__ __device__ functions so that the SAME code is (a) inlined into the
// kernels by nvcc and (b) compiled by g++ (csrc/tests/optim_emu_test.cc checks SGD and AdamW against long-double
// references), without a GPU.  Every product that feeds a sum is an explicit fmaf, so nvcc's contraction and g++'s
// lack of it cannot make the two builds round differently.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define BNET_OPT_HD __host__ __device__ __forceinline__
#else
#define BNET_OPT_HD inline
#endif

namespace bnet {
namespace optim {

// One element of torch.optim.SGD with momentum and L2 weight decay (dampening 0, no Nesterov):
//   d_p = grad*gscale + wd*p;  buf = mu*buf + d_p;  p -= lr*buf
// torch skips the terms of a zero hyper-parameter: with wd == 0 it does not read p, and with mu == 0 it keeps no
// buffer and steps with d_p alone.  So does this: once an infinite gradient has made p or buf infinite, 0 * inf would
// turn every later step of the element into NaN where torch keeps the infinity.  With mu == 0, buf = d_p is still
// stored, so the state layout does not depend on mu.  For finite values the selects change nothing: 0 * x + y == y.
BNET_OPT_HD void sgd_update(float grad, float& p, float& buf, float lr, float mu, float wd, float gscale) {
  const float g = grad * gscale;
  const float dp = wd == 0.0f ? g : fmaf(wd, p, g);
  buf = mu == 0.0f ? dp : fmaf(mu, buf, dp);
  p = fmaf(-lr, buf, p);
}

// Hyper-parameter block of the fused AdamW kernel: 8 floats of device memory, 16-byte aligned, read when the kernel
// runs, so a captured CUDA graph follows a learning-rate schedule and the bias correction without being re-captured.
// `step` counts the steps already taken (the kernel uses t = step + 1).  A float counts exactly up to 2^24 steps.
enum { kHpLr = 0, kHpBeta1, kHpBeta2, kHpEps, kHpWeightDecay, kHpGradScale, kHpStep, kHpReserved, kHpWords };

struct AdamWCoef {
  float decay;       // 1 - lr * weight_decay
  float beta1, omb1; // beta1, 1 - beta1
  float beta2, omb2; // beta2, 1 - beta2
  float step_size;   // lr / (1 - beta1^t)
  float bc2_sqrt;    // sqrt(1 - beta2^t)
  float eps, gscale;
};

// The bias corrections are taken in double: 1 - beta2^t at t = 1 is a difference of nearly equal numbers, and
// fp32 powf would cost it up to ~1e-4 of relative accuracy.  This runs once per thread, not per element.
BNET_OPT_HD AdamWCoef adamw_coef(const float* hp) {
  AdamWCoef c;
  const double lr = hp[kHpLr], b1 = hp[kHpBeta1], b2 = hp[kHpBeta2];
  const double t = (double)hp[kHpStep] + 1.0;
  c.decay = (float)(1.0 - lr * (double)hp[kHpWeightDecay]);
  c.beta1 = hp[kHpBeta1];
  c.omb1 = (float)(1.0 - b1);
  c.beta2 = hp[kHpBeta2];
  c.omb2 = (float)(1.0 - b2);
  c.step_size = (float)(lr / (1.0 - pow(b1, t)));
  c.bc2_sqrt = (float)sqrt(1.0 - pow(b2, t));
  c.eps = hp[kHpEps];
  c.gscale = hp[kHpGradScale];
  return c;
}

// One element of torch.optim.AdamW (amsgrad=False, maximize=False), in the order of torch's fused CUDA kernel:
//   g = grad * gscale;  p *= 1 - lr*wd;  m = b1*m + (1-b1)*g;  v = b2*v + (1-b2)*g*g;
//   p -= step_size * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// IEEE arithmetic carries NaN and Inf where torch's does: a NaN gradient makes this element's p, m and v NaN; an
// infinite one makes m and v infinite and p NaN (inf / inf).  |g| beyond ~1.8e19 overflows g*g in fp32, as it does
// in torch's fp32 state.
BNET_OPT_HD void adamw_update(float grad, float& p, float& m, float& v, const AdamWCoef& c) {
  const float g = grad * c.gscale;
  p = p * c.decay;
  m = fmaf(c.beta1, m, c.omb1 * g);
  v = fmaf(c.beta2, v, (c.omb2 * g) * g);
  const float denom = sqrtf(v) / c.bc2_sqrt + c.eps;
  p = fmaf(-c.step_size, m / denom, p);
}

// Gradient clipping by global norm, as torch.nn.utils.clip_grad_norm_(norm_type=2, error_if_nonfinite=False):
//   clip_coef = clamp(max_norm / (total_norm + 1e-6), max=1)
// in fp32, like torch's fp32 norm tensor.  clamp propagates NaN and fminf(1, NaN) does not, so the clamp is a compare
// that is false for NaN: a NaN norm gives a NaN coefficient.  An infinite norm gives 0 (and an infinite gradient
// element times 0 gives NaN), max_norm = inf with a finite norm gives 1.
BNET_OPT_HD float clip_coef(float max_norm, float total_norm) {
  const float c = max_norm / (total_norm + 1e-6f);
  return c > 1.0f ? 1.0f : c;
}

// Device block of the clipped step (separate from the optimizers' hyper-parameter blocks): 4 floats, 16-byte aligned.
// max_norm is written by the host; the norm kernel writes total_norm (before clipping) and clip_coef every step.
enum { kClipMaxNorm = 0, kClipTotalNorm, kClipCoef, kClipReserved, kClipWords };

// LARS trust ratio of one tensor, as NVIDIA Apex's LARC (clip=False) computes it from the tensor's weight norm wn and
// gradient norm gn:  t = eta * wn / (gn + wd * wn + eps),  and t = 1 when wn == 0 or gn == 0.  The tests are == 0 as
// in Apex, so a NaN norm gives a NaN ratio (the tensor is poisoned, as in the reference) and gn = inf gives t = 0.
BNET_OPT_HD float lars_trust(float eta, float eps, float wd, float wn, float gn) {
  if (wn == 0.0f || gn == 0.0f) return 1.0f;
  return eta * wn / (fmaf(wd, wn, gn) + eps);
}

// One tensor's LARS step as update scalars for sgd_update (with the tensor's gradient already summed over ranks):
// gscale = grad_scale * clip_coef * t and wd = weight_decay * t, so that buf = mu*buf + t*(g + wd*p) up to rounding.
// Excluded tensors (biases, normalisation weights) take t = 1 and no weight decay.  When either norm is 0, Apex's LARC
// leaves the gradient alone -- t = 1 and no weight decay either -- and so does this.
struct LarsScalars {
  float t, gscale, wd;
};
BNET_OPT_HD LarsScalars lars_scalars(float eta, float eps, float wd, float gs, float wn, float gn, bool excluded) {
  if (excluded || wn == 0.0f || gn == 0.0f) return {1.0f, gs, 0.0f};
  const float t = lars_trust(eta, eps, wd, wn, gn);
  return {t, gs * t, wd * t};
}

// Hyper-parameter block of the LARS step: 8 floats of device memory, 16-byte aligned, read when the kernels run.
// The first four are the SGD block's {lr, momentum, weight_decay, grad_scale}.
enum { kLarsLr = 0, kLarsMomentum, kLarsWeightDecay, kLarsGradScale, kLarsEta, kLarsEps, kLarsReserved0, kLarsReserved1,
       kLarsWords };

// Parameter groups: the group table has one row of 4 floats per group, {lr, weight_decay, reserved, reserved}, and a
// bucket's segment table per rank has int rows {vec0, nvec, group, reserved} (BnetGroupSeg), sorted by vec0, the first at
// vector 0, covering the shard exactly once.  `seg` points at the first row's vec0; rows are 4 ints apart.  A shard has
// fewer than 2^31 vectors (the host checks it), so vector indices are ints.
enum { kGroupLr = 0, kGroupWeightDecay, kGroupReserved0, kGroupReserved1, kGroupWords };

// The row holding shard vector v: the last row whose vec0 <= v (binary search; row 0 starts at 0).
BNET_OPT_HD int group_seg_find(const int* seg, int nseg, int v) {
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int m = (lo + hi + 1) >> 1;
    if (seg[4 * m] <= v) lo = m;
    else hi = m - 1;
  }
  return lo;
}

// The same row, found by walking forward from row c, which holds a vector <= v.  A thread's vectors only increase, so a
// cursor kept across them walks every row at most once in all.
BNET_OPT_HD int group_seg_advance(const int* seg, int nseg, int c, int v) {
  while (c + 1 < nseg && seg[4 * (c + 1)] <= v) ++c;
  return c;
}

// Device block of the exponential moving average of the master weights: 4 floats, 16-byte aligned.  `weight` is
// 1 - decay, computed in double by the host and rounded once, which is the fp32 weight torch._foreach_lerp_ gets from
// torch.optim.swa_utils.get_ema_multi_avg_fn(decay).  `step` counts the optimizer steps taken and `n_averaged` the EMA
// updates, as AveragedModel.n_averaged; both are advanced on the device (bnet_ema_advance_kernel), so a captured CUDA
// graph keeps counting.  A float counts exactly up to 2^24 steps.
enum { kEmaWeight = 0, kEmaEvery, kEmaStep, kEmaNAveraged, kEmaWords };

// Whether the optimizer step about to be counted (step + 1, steps counted from 1) updates the EMA, and whether that
// update is a copy (no update averaged yet, as AveragedModel's n_averaged == 0).  `every` >= 1.
struct EmaGate {
  bool update, copy;
};
BNET_OPT_HD EmaGate ema_gate(float step, float every, float n_averaged) {
  const bool update = ((unsigned)step + 1u) % (unsigned)every == 0u;
  return {update, update && n_averaged == 0.0f};
}

// torch.lerp(ema, w, weight) in fp32: ema + weight*(w - ema) for |weight| < 0.5, else w - (w - ema)*(1 - weight).  The
// second branch makes weight = 1 give w exactly.  NaN and Inf follow IEEE arithmetic as in torch's kernel: a NaN in
// either operand gives NaN, and ema = +-Inf with w finite gives NaN (Inf - Inf) in the first branch.
BNET_OPT_HD float ema_lerp(float ema, float w, float weight) {
  const float d = w - ema;
  return fabsf(weight) < 0.5f ? fmaf(weight, d, ema) : fmaf(-d, 1.0f - weight, w);
}

}  // namespace optim
}  // namespace bnet

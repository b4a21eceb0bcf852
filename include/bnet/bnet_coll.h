/*
 * bnet collectives — extension API over symmetric (peer-mapped) GPU memory.
 *
 * The reference moves bytes for NCCL and leaves the reduction to NCCL's kernels
 * (SURVEY.md §2.5, K4-K6 in §2.6).  On an NVSwitch box the transport and the
 * reduction fuse: these entry points run hand-written sm_90a kernels that reduce
 * in the switch (NVLS multimem.ld_reduce / multimem.st on a cuMulticast mapping) or
 * with peer loads/stores over NVLink, optionally fused with the optimizer step.
 *
 * Setup is staged so that a host-side communicator (torch.distributed, MPI, …) can
 * carry the small handshake blobs between ranks:
 *   create -> export(blob) -> [all_gather blobs] -> import(blobs)
 *          -> mc_add_device -> [barrier] -> mc_bind -> [barrier]
 */
#ifndef BNET_COLL_H_
#define BNET_COLL_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BNET_COLL_BLOB_BYTES 128
#define BNET_COLL_MAX_WORLD 16
#define BNET_COLL_MAX_BLOCKS 304
#define BNET_COLL_CHANNELS 8
#define BNET_COLL_SIGNAL_BYTES (BNET_COLL_CHANNELS * BNET_COLL_MAX_BLOCKS * BNET_COLL_MAX_WORLD * 4)

typedef struct BnetColl BnetColl;

enum { BNET_F32 = 0, BNET_BF16 = 1, BNET_F16 = 2 };
enum { BNET_SUM = 0, BNET_AVG = 1, BNET_MAX = 2, BNET_MIN = 3 };
enum {
  BNET_ALGO_AUTO = 0,
  BNET_ALGO_NVLS = 1,       /* multimem.ld_reduce + multimem.st, in place                 */
  BNET_ALGO_P2P_TWOSHOT = 2, /* reduce-scatter with peer loads, all-gather with peer stores */
  BNET_ALGO_P2P_ONESHOT = 3  /* every rank reads every peer; latency-optimal, out of place  */
};

int bnet_coll_create(int rank, int world, int dev, size_t heap_bytes, BnetColl** out);
int bnet_coll_export(BnetColl* c, void* blob);                 /* BNET_COLL_BLOB_BYTES */
int bnet_coll_import(BnetColl* c, const void* blobs);          /* world * BNET_COLL_BLOB_BYTES */
int bnet_coll_mc_add_device(BnetColl* c);                      /* no-op without multicast */
int bnet_coll_mc_bind(BnetColl* c);
int bnet_coll_destroy(BnetColl* c);

void* bnet_coll_heap(BnetColl* c);            /* local VA of the symmetric heap (after the signal pad) */
size_t bnet_coll_heap_bytes(BnetColl* c);
void* bnet_coll_peer_heap(BnetColl* c, int peer);
void* bnet_coll_mc_heap(BnetColl* c);         /* multicast VA or NULL */
int bnet_coll_has_multicast(BnetColl* c);
const char* bnet_coll_last_error(void);

/* In-place all-reduce of `count` elements at byte `offset` of the heap (same offset on every rank).
 * offset and count*elsize must be multiples of 16*world.  Launches on `stream`; returns the number of
 * kernels launched (>0) or <0 on error. */
int bnet_allreduce(BnetColl* c, size_t offset, size_t count, int dtype, int op, int algo, int channel,
                   int nblocks, void* stream);
/* Out-of-place one-shot variant: result written to local pointer `out`. */
int bnet_allreduce_oneshot(BnetColl* c, size_t offset, void* out, size_t count, int dtype, int op, int channel,
                           int nblocks, void* stream);
/* Latency-optimal small all-reduce: no barrier, the flag travels inside every 8-byte word ("LL").  `ll_offset` names an
 * area of bnet_allreduce_ll_area_bytes(world, ll_words) bytes in the heap (zero before the first use, same offset on
 * every rank, used by nothing else); every rank makes the same sequence of calls on it (the call counter that serves
 * as the flag lives in the area itself, so a captured CUDA graph replays correctly).  in / out are ordinary local device
 * pointers (in place allowed), count * elsize <= 4 * ll_words. */
size_t bnet_allreduce_ll_area_bytes(int world, size_t ll_words);
int bnet_allreduce_ll(BnetColl* c, size_t ll_offset, size_t ll_words, const void* in, void* out, size_t count, int dtype,
                      int op, void* stream);
int bnet_barrier(BnetColl* c, int channel, void* stream);

/* Fused gradient all-reduce + SGD(momentum, weight decay) + parameter broadcast (one kernel):
 *   g     = mean over ranks of grad[bucket]           (in-switch or peer-load reduction)
 *   owner : buf = mu*buf + g + wd*p ; p -= lr*buf     (fp32 master + momentum, sharded 1/world)
 *   param[bucket] on EVERY rank <- p                  (multimem.st / peer stores)
 *   grad[bucket] <- 0 when zero_grads                 (ready for the next in-place accumulation)
 * grad_off/param_off: byte offsets in the heap; count elements of `dtype`, multiple of 8*world.
 * master/momentum: local fp32 arrays of count/world elements (this rank's shard). */
int bnet_fused_allreduce_sgd(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype, float lr,
                             float momentum, float weight_decay, float grad_scale, float* master, float* mom_buf,
                             int zero_grads, int channel, int nblocks, void* stream);
/* Same, with {lr, momentum, weight_decay, grad_scale} read from 4 floats of device memory (16-byte aligned) when the
 * kernel runs: a captured CUDA graph follows a learning-rate schedule without being re-captured. */
int bnet_fused_allreduce_sgd_hp(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype, const float* hp_dev,
                                float* master, float* mom_buf, int zero_grads, int channel, int nblocks, void* stream);
/* Fused gradient all-reduce + AdamW (decoupled weight decay, torch.optim.AdamW semantics without amsgrad / maximize) +
 * parameter broadcast, one kernel, laid out like bnet_fused_allreduce_sgd.  Per element of the owner's shard, with
 * g = sum over ranks of grad * grad_scale and t = step + 1:
 *   p = p*(1 - lr*wd);  m = b1*m + (1-b1)*g;  v = b2*v + (1-b2)*g*g;  p -= lr/(1-b1^t) * m / (sqrt(v)/sqrt(1-b2^t) + eps)
 * hp_dev: 8 floats of device memory, 16-byte aligned, read when the kernel runs:
 *   {lr, beta1, beta2, eps, weight_decay, grad_scale, step, reserved}
 * `step` is the number of steps already taken; the caller advances it once per training step (not per bucket), so a
 * captured CUDA graph follows the schedule and the bias correction.  A float counts steps exactly up to 2^24.
 * master/exp_avg/exp_avg_sq: local fp32 arrays of count/world elements (this rank's shard), 16-byte aligned. */
int bnet_fused_allreduce_adamw(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype, const float* hp_dev,
                               float* master, float* exp_avg, float* exp_avg_sq, int zero_grads, int channel, int nblocks,
                               void* stream);

/* Fused step with gradient clipping by global L2 norm (torch.nn.utils.clip_grad_norm_, norm type 2), in three stages on
 * one stream.  The clip block is 4 floats of device memory, 16-byte aligned: {max_norm, total_norm, clip_coef, reserved};
 * the caller writes max_norm, stage 2 writes the other two every step.
 *
 * Stage 1, per bucket: reduce the bucket's gradients over the ranks like bnet_fused_allreduce_sgd, but store this rank's
 * shard of the sum as fp32 in `scratch` (count/world floats, 16-byte aligned) instead of updating, write the sum of squares
 * of each CTA's share (in double) to its slot of the `partial` row (BNET_COLL_CLIP_ROW doubles; slots beyond the grid are
 * zeroed), and zero grad[bucket].  Deterministic: no atomics, the same grid gives the same bits. */
#define BNET_COLL_CLIP_ROW BNET_COLL_MAX_BLOCKS
int bnet_fused_clip_reduce_norm(BnetColl* c, size_t grad_off, size_t count, int dtype, float* scratch, double* partial,
                                int channel, int nblocks, void* stream);
/* Stage 1 of a micro-batch that accumulates (gradient accumulation, every micro-batch after the bucket's first in the
 * step): the same reduction and checks, but scratch[i] = scratch[i] + sum (fp32), the partial row gets the sums of
 * squares of the NEW scratch values, and grad[bucket] is zeroed.  Same determinism. */
int bnet_fused_accum_reduce_norm(BnetColl* c, size_t grad_off, size_t count, int dtype, float* scratch, double* partial,
                                 int channel, int nblocks, void* stream);
/* Stage 2, once per step after every bucket's stage 1 (and after the caller's stream has waited for backward): sum the
 * nrows x BNET_COLL_CLIP_ROW doubles at `partials` in a fixed order, exchange the per-rank sums through `world` doubles at
 * heap byte offset `xchg_off` (16-byte aligned, same offset on every rank, used by nothing else) and add them in rank
 * order, so every rank gets the same bits; then total_norm = sqrt(sum) * grad_scale and
 * clip_coef = clamp(max_norm / (total_norm + 1e-6), max=1) (NaN propagates).  One CTA, two rank barriers. */
int bnet_fused_clip_coef(BnetColl* c, const double* partials, int nrows, size_t xchg_off, float grad_scale, float* clip,
                         int channel, void* stream);
/* Stage 3, per bucket after stage 2: the SGD or AdamW update of bnet_fused_allreduce_sgd[_hp] / _adamw with the gradient
 * scratch[i] * clip_coef in place of the rank-summed gradient, then the parameter broadcast and a closing barrier.  No
 * gradient zeroing (stage 1 did it).  With max_norm = inf and a finite norm, clip_coef is 1 and the result is bitwise the
 * one-kernel step's. */
int bnet_fused_clip_apply_sgd(BnetColl* c, size_t param_off, size_t count, int dtype, const float* scratch, const float* clip,
                              float lr, float momentum, float weight_decay, float grad_scale, float* master, float* mom_buf,
                              int channel, int nblocks, void* stream);
int bnet_fused_clip_apply_sgd_hp(BnetColl* c, size_t param_off, size_t count, int dtype, const float* scratch,
                                 const float* clip, const float* hp_dev, float* master, float* mom_buf, int channel, int nblocks,
                                 void* stream);
int bnet_fused_clip_apply_adamw(BnetColl* c, size_t param_off, size_t count, int dtype, const float* scratch, const float* clip,
                                const float* hp_dev, float* master, float* exp_avg, float* exp_avg_sq, int channel, int nblocks,
                                void* stream);

/* LARS (layer-wise adaptive rate scaling, NVIDIA Apex LARC with clip=False, then SGD with momentum) in the staged step.
 * Stage 1 is bnet_fused_clip_reduce_norm / bnet_fused_accum_reduce_norm as above.  Each parameter tensor's update takes a
 * trust ratio from the norms of the WHOLE tensor, so three more launches follow, on the same stream:
 *
 * A segment is the part of one parameter tensor that lies in this rank's shard of a bucket: `nvec` 16-byte vectors from
 * shard vector `vec0` (every tensor starts on a 16-byte boundary, so a vector belongs to one tensor; zero padding
 * vectors may belong to either neighbouring segment).  A bucket's table lists its segments sorted by vec0 and covers
 * the shard exactly once.  Each segment is cut into chunks of BNET_LARS_CHUNK vectors, and chunk k of a segment owns
 * norm slot `slot0 + k` (slot0 is a running count over the bucket's segments).  The caller validates the tables before
 * it uploads them: the kernels trust them. */
#define BNET_LARS_CHUNK 4096
typedef struct {
  int32_t vec0, nvec, tensor, slot0;
} BnetLarsSeg;
/* Per tensor, for the trust kernel: its norm slots [slot0, slot0 + nslots) in the slot array of all buckets (nslots = 0
 * when no part of it is in this rank's shards); `excluded` != 0 for tensors that take no trust ratio or weight decay. */
typedef struct {
  int32_t slot0, nslots, excluded, reserved;
} BnetLarsTensor;
/* Per bucket, once per step after stage 1: for each chunk of each segment, the sums of squares (in double, fixed order,
 * no atomics: the bits depend on neither the grid nor the repeat) of this rank's fp32 `master` and `scratch` shard
 * (count/world floats each) into slots[2 * slot] = sum w^2 and slots[2 * slot + 1] = sum g^2.  Rank-local. */
int bnet_fused_lars_norm(BnetColl* c, size_t count, int dtype, const float* master, const float* scratch,
                         const BnetLarsSeg* segs, int nseg, double* slots, int nslots, int nblocks, void* stream);
/* Once per step, after every norm launch (and after bnet_fused_clip_coef when clipping; its barrier then is the
 * step's): per tensor, sum its slots, exchange the per-rank (sum w^2, sum g^2) through 2 * world * ntensors doubles at
 * heap byte offset `xchg_off` (16-byte aligned, same on every rank, used by nothing else) and add them in rank order, so
 * every rank gets the same bits; then wn = sqrt(w^2), gn = sqrt(g^2) * grad_scale * clip_coef,
 * t = lars_trust(eta, eps, wd, wn, gn) (csrc/cuda/optim_body.cuh), and the tensor's update scalars
 * scal[2j] = grad_scale * clip_coef * t, scal[2j + 1] = wd * t (excluded: grad_scale * clip_coef and 0, t = 1), and
 * trust[j] = t.  `clip`: the 4-float clip block (clip_coef read from it); `hp`: the 8-float LARS block
 * {lr, momentum, weight_decay, grad_scale, trust_coefficient, eps, reserved, reserved}.  One CTA, two rank barriers. */
int bnet_fused_lars_trust(BnetColl* c, const double* slots, const BnetLarsTensor* tensors, int ntensors, size_t xchg_off,
                          const float* clip, const float* hp, float* scal, float* trust, int channel, void* stream);
/* Per bucket after the trust kernel: the SGD update of bnet_fused_clip_apply_sgd_hp from `scratch`, with every vector's
 * gradient scale and weight decay taken from its tensor's scal pair (lr and momentum from hp), then the parameter
 * broadcast and a closing barrier. */
int bnet_fused_lars_apply(BnetColl* c, size_t param_off, size_t count, int dtype, const float* scratch, const BnetLarsSeg* segs,
                          int nseg, const float* scal, const float* hp, float* master, float* mom_buf, int channel, int nblocks,
                          void* stream);

/* Parameter groups: the SGD and AdamW steps with a learning rate and weight decay per group of parameter tensors, as
 * torch.optim's param groups.  The group table is `ngroups` rows of 4 floats of device memory, 16-byte aligned:
 * {lr, weight_decay, reserved, reserved} (csrc/cuda/optim_body.cuh), read when the kernel runs, so a captured CUDA graph
 * follows changes to it; 1 <= ngroups <= BNET_GROUPS_MAX.
 *
 * A group segment is a run of consecutive shard vectors of one group: `nvec` 16-byte vectors from shard vector `vec0`.
 * A bucket's table per rank lists them sorted by vec0 and covers the shard exactly once; every tensor starts on a 16-byte
 * boundary, so no vector holds two tensors, and zero padding joins a neighbouring segment.  The caller validates the
 * table (group indices below ngroups included) before it uploads it: the kernels trust it. */
#define BNET_GROUPS_MAX 64
typedef struct {
  int32_t vec0, nvec, group, reserved;
} BnetGroupSeg;
/* bnet_fused_allreduce_sgd_hp with every vector's lr and weight decay taken from its group's row: the momentum and
 * grad_scale come from the 4-float SGD block hp_dev, whose lr and weight_decay are not read.  A group with weight decay 0
 * skips the decay term, as torch does. */
int bnet_fused_allreduce_sgd_groups(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype, const float* hp_dev,
                                    const float* groups, int ngroups, const BnetGroupSeg* segs, int nseg, float* master,
                                    float* mom_buf, int zero_grads, int channel, int nblocks, void* stream);
/* bnet_fused_allreduce_adamw with every vector's lr and weight decay taken from its group's row; betas, eps, grad_scale and
 * step come from the 8-float AdamW block hp_dev, whose lr and weight_decay are not read.  A group's elements get the bits
 * the ungrouped kernel gives them with the group's lr and weight decay in the block. */
int bnet_fused_allreduce_adamw_groups(BnetColl* c, size_t grad_off, size_t param_off, size_t count, int dtype, const float* hp_dev,
                                      const float* groups, int ngroups, const BnetGroupSeg* segs, int nseg, float* master,
                                      float* exp_avg, float* exp_avg_sq, int zero_grads, int channel, int nblocks, void* stream);
/* Stage 3 of the staged step with groups: bnet_fused_clip_apply_sgd_hp / _adamw with the per-group values as above. */
int bnet_fused_clip_apply_sgd_groups(BnetColl* c, size_t param_off, size_t count, int dtype, const float* scratch, const float* clip,
                                     const float* hp_dev, const float* groups, int ngroups, const BnetGroupSeg* segs, int nseg,
                                     float* master, float* mom_buf, int channel, int nblocks, void* stream);
int bnet_fused_clip_apply_adamw_groups(BnetColl* c, size_t param_off, size_t count, int dtype, const float* scratch,
                                       const float* clip, const float* hp_dev, const float* groups, int ngroups,
                                       const BnetGroupSeg* segs, int nseg, float* master, float* exp_avg, float* exp_avg_sq,
                                       int channel, int nblocks, void* stream);

/* Exponential moving average (EMA) of the fp32 master weights, as torch.optim.swa_utils.AveragedModel with
 * get_ema_multi_avg_fn(decay) and use_buffers=False, applied to this rank's master shards.  The EMA block is 4 floats of
 * device memory, 16-byte aligned: {weight = 1 - decay, every, step, n_averaged} (csrc/cuda/optim_body.cuh).  `step`
 * counts the optimizer steps taken; step s (counted from 1) is an EMA step when s % every == 0.  Counters are floats,
 * exact up to 2^24.
 *
 * Per bucket, after the optimizer step's last update: on an EMA step, ema = master when n_averaged == 0, else
 * ema = torch.lerp(ema, master, weight), over `count` floats (a whole number of float4s, both shards 16-byte aligned);
 * on any other step the kernel reads the block and exits.  Rank-local, deterministic, no barriers. */
int bnet_ema_update(BnetColl* c, size_t count, const float* master, float* ema, const float* blk, int nblocks, void* stream);
/* Once per optimizer step, after every bucket's bnet_ema_update: n_averaged += 1 on an EMA step, then step += 1.  One
 * thread. */
int bnet_ema_advance(BnetColl* c, float* blk, void* stream);

/* Multi-tensor pack+cast into the heap (K5): n tensors described on the device. */
typedef struct {
  const void* src;
  uint64_t dst_elem_off;   /* element offset inside the destination flat buffer */
  uint64_t numel;
} BnetPackItem;
int bnet_pack_cast(const BnetPackItem* items_dev, int n, void* dst, int src_dtype, int dst_dtype, float scale,
                   uint64_t max_numel, void* stream);

#ifdef __cplusplus
}
#endif
#endif

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

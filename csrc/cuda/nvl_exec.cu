// sm_90a copy/reduce executor behind the NVLink transport's isend (K1, K4, K5, K7,
// K8 of SURVEY.md §2.6).
//
// One "device stream" = one thread-block cluster running a semi-persistent kernel
// that pulls work descriptors from a ring in pinned host memory — the device-side
// analogue of the reference's per-TCP-stream worker thread + channel
// (reference: nthread_…:336-361).  The host dispatcher splits a message into
// max(ceil(n/nclusters), MIN_CHUNKSIZE)-byte chunks and deals them round-robin to
// the clusters, cursor persisting across messages (reference: nthread_…:393-413).
//
// Inside a cluster: the leader CTA polls the ring (ld.acquire.sys on host memory),
// broadcasts the descriptor through distributed shared memory, all CTAs move their
// share with 16-byte vector loads/stores (or a TMA bulk-copy pipeline, UBLKCP,
// when BNET_COPY_ENGINE=tma) straight into the peer GPU's buffer over NVLink,
// optionally fused with an accumulate (red.global.add) or a bf16<->fp32 cast, then
// a cluster barrier, a system-scope fence and a release store of the chunk's
// completion word (pinned host memory, polled by test()).
//
// The kernel parks with nanosleep back-off while idle and leaves after
// BNET_KERNEL_IDLE_US without work so that cudaDeviceSynchronize()/cudaFree() in
// the application never wait on us for long; the host relaunches on demand with a
// Dekker-style handshake on the queue's state word.
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <mutex>

#include "core/common.h"
#include "cuda/cuda_iface.h"
#include "cuda/driver_api.h"
#include "cuda/exec_body.cuh"
#include "cuda/nvl_exec.h"
#include "cuda/ptx.cuh"

namespace bnet {
namespace cuda {

constexpr int kQueueDepth = 64;
constexpr int kThreads = 512;
constexpr uint32_t ST_EXITED = 0, ST_RUNNING = 1, ST_EXITING = 2;

struct alignas(64) Desc {
  uint64_t seq;        // == index+1 when valid (written last, release)
  const void* src;
  void* dst;
  uint64_t nbytes;     // bytes of SOURCE to process
  uint64_t* flag;      // device-visible completion word (pinned host memory)
  uint64_t flag_val;
  uint32_t op;
  float scale;         // fp8 (de)quantisation scale
};

struct ClusterQ {
  alignas(64) volatile uint64_t tail;    // host: descriptors published
  alignas(64) volatile uint64_t head;    // device: descriptors completed
  alignas(64) volatile uint32_t state;   // ST_*
  alignas(64) volatile uint32_t stop;    // host asks the kernel to leave
  alignas(64) volatile uint64_t err;     // device reports a watchdog trip
  alignas(64) Desc d[kQueueDepth];
};

// ------------------------------------------------------------------ device code
struct SmemDesc {
  const char* src;
  char* dst;
  uint64_t nbytes;
  uint32_t op;
  uint32_t quit;
  float scale;
  uint32_t pad;
};

// TMA bulk-copy pipeline: one elected thread per CTA moves its share through a ring of
// shared-memory stages with cp.async.bulk (global->shared, shared->peer global).
constexpr int kTmaStages = 4;
constexpr uint32_t kTmaStageBytes = 32768;

__device__ void tma_copy_range(const char* src, char* dst, size_t n, char* smem, uint64_t* bars, uint32_t* phases) {
  // n, src, dst are multiples of 16 here (checked by the caller)
  const size_t nchunks = (n + kTmaStageBytes - 1) / kTmaStageBytes;
  constexpr int D = kTmaStages - 1;   // loads in flight ahead of the store front
  auto bytes_of = [&](size_t i) -> uint32_t {
    size_t off = i * (size_t)kTmaStageBytes;
    return (uint32_t)(n - off < kTmaStageBytes ? n - off : kTmaStageBytes);
  };
  auto issue_load = [&](size_t i) {
    int s = (int)(i % kTmaStages);
    uint32_t b = bytes_of(i);
    ptx::mbar_arrive_expect_tx(&bars[s], b);
    ptx::bulk_g2s(smem + (size_t)s * kTmaStageBytes, src + i * (size_t)kTmaStageBytes, b, &bars[s]);
  };
  for (size_t i = 0; i < nchunks && i < (size_t)D; i++) issue_load(i);
  for (size_t i = 0; i < nchunks; i++) {
    int s = (int)(i % kTmaStages);
    ptx::mbar_wait(&bars[s], phases[s]);
    phases[s] ^= 1;
    ptx::bulk_s2g(dst + i * (size_t)kTmaStageBytes, smem + (size_t)s * kTmaStageBytes, bytes_of(i));
    ptx::bulk_commit();
    size_t j = i + D;
    if (j < nchunks) {
      ptx::bulk_wait_read<1>();   // the store issued one iteration ago has drained its stage
      issue_load(j);
    }
  }
  ptx::bulk_wait_all();           // stores performed before we signal completion
}

template <bool kUseTma>
__global__ void __launch_bounds__(kThreads, 1)
bnet_nvl_stream_kernel(ClusterQ* q, uint64_t idle_ns, uint64_t first_idle_ns, const uint32_t* outstanding) {
  extern __shared__ __align__(128) unsigned char dyn_smem[];
  __shared__ SmemDesc sd;
  __shared__ __align__(8) uint64_t bars[kTmaStages];
  __shared__ uint32_t phases[kTmaStages];

  const uint32_t crank = ptx::cluster_ctarank();
  const uint32_t csize = ptx::cluster_nctarank();
  const int tid = threadIdx.x;
  if (kUseTma && tid == 0) {
    for (int s = 0; s < kTmaStages; s++) {
      ptx::mbar_init(&bars[s], 1);
      phases[s] = 0;
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  uint64_t head = q->head;            // same value in every CTA of the cluster
  uint64_t last_work = ptx::globaltimer();
  // armed at connection setup: wait longer for the FIRST job so that it needs no launch on the
  // data path (a launch can be held up by a cudaFree elsewhere in the process: tools/blocking_calls_probe.py)
  uint64_t idle_limit = first_idle_ns > idle_ns ? first_idle_ns : idle_ns;
  for (;;) {
    // ---- leader: wait for the next descriptor, publish it to every CTA of the cluster
    if (crank == 0 && tid == 0) {
      SmemDesc loc;
      loc.quit = 0;
      loc.pad = 0;
      uint32_t backoff = 32;
      Desc* d = &q->d[head % kQueueDepth];
      for (;;) {
        if (ptx::ld_acquire_sys_u64(&d->seq) == head + 1) break;
        uint64_t now = ptx::globaltimer();
        if (ptx::ld_relaxed_sys_u32((const uint32_t*)&q->stop)) { loc.quit = 1; break; }
        // stay resident while the host still has requests in flight on ANY NVL comm of this process (a
        // collective is running: leaving now would force a launch on the data path later); hard cap 10 s
        if (now - last_work > idle_limit &&
            (ptx::ld_relaxed_sys_u32(outstanding) == 0 || now - last_work > 10000000000ull)) {
          // leave unless the host published work while we were deciding (store, fence, re-check)
          ptx::st_release_sys_u32((uint32_t*)&q->state, ST_EXITING);
          ptx::fence_sc_sys();
          if (ptx::ld_acquire_sys_u64(&d->seq) == head + 1) {
            ptx::st_release_sys_u32((uint32_t*)&q->state, ST_RUNNING);
            break;
          }
          loc.quit = 1;
          break;
        }
        __nanosleep(backoff);
        if (backoff < 1024) backoff <<= 1;
      }
      if (!loc.quit) {
        loc.src = (const char*)d->src;
        loc.dst = (char*)d->dst;
        loc.nbytes = d->nbytes;
        loc.op = d->op;
        loc.scale = d->scale;
      } else {
        loc.src = nullptr; loc.dst = nullptr; loc.nbytes = 0; loc.op = 0; loc.scale = 1.0f;
      }
      for (uint32_t r = 0; r < csize; r++) ptx::st_dsmem(&sd, r, loc);   // distributed shared memory broadcast
    }
    ptx::cluster_sync();     // release/acquire at cluster scope; also drops stale L1 lines
    const SmemDesc cur = sd;
    if (cur.quit) break;

    if (cur.op != OP_FLUSH) {
      // ---- every CTA takes a contiguous 16-byte aligned share of the source range
      size_t b0, b1;
      cta_share(cur.op, cur.nbytes, crank, csize, &b0, &b1);
      const char* s = cur.src + b0;
      char* dd = cur.dst + dst_offset_for(cur.op, b0);
      size_t n = b1 - b0;
      bool tma_ok = kUseTma && cur.op == OP_COPY && n >= 16 &&
                    ((((uintptr_t)s | (uintptr_t)dd) & 15) == 0);
      if (tma_ok) {
        size_t nb = n & ~(size_t)15;
        if (tid == 0) tma_copy_range(s, dd, nb, (char*)dyn_smem, bars, phases);
        if (n > nb) process_range(OP_COPY, s + nb, dd + nb, n - nb, tid, kThreads);
      } else {
        process_range(cur.op, s, dd, n, tid, kThreads, cur.scale);
      }
    }
    __syncthreads();
    ptx::cluster_sync();     // every CTA's stores are ordered before the leader's fence
    if (crank == 0 && tid == 0) {
      Desc* d = &q->d[head % kQueueDepth];
      uint64_t* flag = d->flag;
      uint64_t fv = d->flag_val;
      ptx::fence_acq_rel_sys();                    // peer stores visible system-wide ...
      ptx::st_release_sys_u64(flag, fv);           // ... before the chunk's completion word
      ptx::st_release_sys_u64((uint64_t*)&q->head, head + 1);
      last_work = ptx::globaltimer();
      idle_limit = idle_ns;
    }
    head++;
  }
  if (crank == 0 && tid == 0) ptx::st_release_sys_u32((uint32_t*)&q->state, ST_EXITED);
}

// ---- single-grid variant (BNET_EXEC_GRID=1) ------------------------------------------------------------------
// The same per-cluster descriptor queues, but ALL clusters are one grid on ONE stream: a (re)launch is one
// driver call instead of nclusters, and the executor occupies one hardware work queue instead of one per
// cluster (other streams of the process cannot end up queued behind a resident kernel of ours).
// Leaving is a grid-wide decision taken by cluster 0's leader: nothing submitted that is not completed
// (host counter vs device counter), idle for long enough, no request in flight on any comm.  The Dekker
// handshake is the same as above with ctl->submitted in the role of the descriptor's seq word.
struct GridCtl {
  alignas(64) volatile uint32_t state;       // ST_*
  alignas(64) volatile uint32_t stop;        // host asks the grid to leave
  alignas(64) volatile uint64_t submitted;   // host: descriptors published on any queue, ever
};
__device__ unsigned long long g_grid_completed;   // device: descriptors completed by any cluster, ever
__device__ unsigned long long g_grid_last_work;   // device: globaltimer of the latest completion
__device__ unsigned long long g_grid_quit_epoch;  // device: launch epoch whose clusters have been told to leave

template <bool kUseTma>
__global__ void __launch_bounds__(kThreads, 1)
bnet_nvl_grid_kernel(GridCtl* ctl, ClusterQ* const* queues, uint64_t epoch, uint64_t idle_ns, uint64_t first_idle_ns,
                     const uint32_t* outstanding) {
  extern __shared__ __align__(128) unsigned char dyn_smem[];
  __shared__ SmemDesc sd;
  __shared__ __align__(8) uint64_t bars[kTmaStages];
  __shared__ uint32_t phases[kTmaStages];

  const uint32_t crank = ptx::cluster_ctarank();
  const uint32_t csize = ptx::cluster_nctarank();
  const uint32_t cid = blockIdx.x / csize;           // which queue this cluster serves
  ClusterQ* q = queues[cid];
  const int tid = threadIdx.x;
  if (kUseTma && tid == 0) {
    for (int s = 0; s < kTmaStages; s++) {
      ptx::mbar_init(&bars[s], 1);
      phases[s] = 0;
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  uint64_t head = q->head;
  const uint64_t t_start = ptx::globaltimer();
  uint64_t idle_limit = first_idle_ns > idle_ns ? first_idle_ns : idle_ns;
  for (;;) {
    if (crank == 0 && tid == 0) {
      SmemDesc loc;
      loc.quit = 0;
      loc.pad = 0;
      uint32_t backoff = 32;
      Desc* d = &q->d[head % kQueueDepth];
      for (;;) {
        if (ptx::ld_acquire_sys_u64(&d->seq) == head + 1) break;
        if (ptx::ld_relaxed_sys_u32((const uint32_t*)&ctl->stop)) { loc.quit = 1; break; }
        if (*(volatile unsigned long long*)&g_grid_quit_epoch == epoch) { loc.quit = 1; break; }
        if (cid == 0) {
          const uint64_t now = ptx::globaltimer();
          uint64_t lw = *(volatile unsigned long long*)&g_grid_last_work;
          if (lw < t_start) lw = t_start;            // completions of earlier launches do not count
          // (globaltimer is read on different SMs: a completion stamped by another cluster may be a few ns "ahead")
          const uint64_t idle = now > lw ? now - lw : 0;
          if (idle > idle_limit && (ptx::ld_relaxed_sys_u32(outstanding) == 0 || idle > 10000000000ull)) {
            ptx::st_release_sys_u32((uint32_t*)&ctl->state, ST_EXITING);
            ptx::fence_sc_sys();
            const uint64_t sub = ptx::ld_acquire_sys_u64((const uint64_t*)&ctl->submitted);
            const uint64_t comp = *(volatile unsigned long long*)&g_grid_completed;
            if (sub != comp) {
              // work was published (or is still running on another cluster) while we were deciding: stay
              ptx::st_release_sys_u32((uint32_t*)&ctl->state, ST_RUNNING);
              idle_limit = idle_ns;
              atomicMax(&g_grid_last_work, (unsigned long long)now);
            } else {
              atomicExch(&g_grid_quit_epoch, (unsigned long long)epoch);   // the other clusters follow
              __threadfence();
              loc.quit = 1;
              break;
            }
          }
        }
        __nanosleep(backoff);
        if (backoff < 1024) backoff <<= 1;
      }
      if (!loc.quit) {
        loc.src = (const char*)d->src;
        loc.dst = (char*)d->dst;
        loc.nbytes = d->nbytes;
        loc.op = d->op;
        loc.scale = d->scale;
      } else {
        loc.src = nullptr; loc.dst = nullptr; loc.nbytes = 0; loc.op = 0; loc.scale = 1.0f;
      }
      for (uint32_t r = 0; r < csize; r++) ptx::st_dsmem(&sd, r, loc);
    }
    ptx::cluster_sync();
    const SmemDesc cur = sd;
    if (cur.quit) break;

    if (cur.op != OP_FLUSH) {
      size_t b0, b1;
      cta_share(cur.op, cur.nbytes, crank, csize, &b0, &b1);
      const char* s = cur.src + b0;
      char* dd = cur.dst + dst_offset_for(cur.op, b0);
      size_t n = b1 - b0;
      bool tma_ok = kUseTma && cur.op == OP_COPY && n >= 16 && ((((uintptr_t)s | (uintptr_t)dd) & 15) == 0);
      if (tma_ok) {
        size_t nb = n & ~(size_t)15;
        if (tid == 0) tma_copy_range(s, dd, nb, (char*)dyn_smem, bars, phases);
        if (n > nb) process_range(OP_COPY, s + nb, dd + nb, n - nb, tid, kThreads);
      } else {
        process_range(cur.op, s, dd, n, tid, kThreads, cur.scale);
      }
    }
    __syncthreads();
    ptx::cluster_sync();
    if (crank == 0 && tid == 0) {
      Desc* d = &q->d[head % kQueueDepth];
      uint64_t* flag = d->flag;
      uint64_t fv = d->flag_val;
      ptx::fence_acq_rel_sys();
      ptx::st_release_sys_u64(flag, fv);
      ptx::st_release_sys_u64((uint64_t*)&q->head, head + 1);
      atomicMax(&g_grid_last_work, (unsigned long long)ptx::globaltimer());
      __threadfence();
      atomicAdd(&g_grid_completed, 1ull);          // after the completion word: "completed" implies "signalled"
      idle_limit = idle_ns;
    }
    head++;
  }
  // cluster 0 took the decision: it is also the one that reports it (the relaunch is stream-ordered behind
  // the clusters that are still on their way out)
  if (cid == 0 && crank == 0 && tid == 0) ptx::st_release_sys_u32((uint32_t*)&ctl->state, ST_EXITED);
}

// One-shot kernel used when BNET_PERSISTENT=0: a grid of clusters per chunk list.
struct OneShotArgs {
  const char* src;
  char* dst;
  uint64_t nbytes;
  uint64_t* flag;
  uint64_t flag_val;
  uint32_t op;
  float scale;
};
__global__ void __launch_bounds__(kThreads, 1) bnet_nvl_oneshot_kernel(OneShotArgs a) {
  const uint32_t crank = ptx::cluster_ctarank();
  const uint32_t csize = ptx::cluster_nctarank();
  if (a.op != OP_FLUSH) {
    size_t b0, b1;
    cta_share(a.op, a.nbytes, crank, csize, &b0, &b1);
    process_range(a.op, a.src + b0, a.dst + dst_offset_for(a.op, b0), b1 - b0, threadIdx.x, kThreads, a.scale);
  }
  __syncthreads();
  ptx::cluster_sync();
  if (crank == 0 && threadIdx.x == 0) {
    ptx::fence_acq_rel_sys();
    ptx::st_release_sys_u64(a.flag, a.flag_val);
  }
}

// ---- per-message kernel: the default behind NCCL's isend (BNET_EXEC_MODE=msg) --------------------------------
// ONE launch moves a whole message: cluster c takes chunk c (the striping rule of the reference, applied to
// clusters), the CTAs of a cluster split the chunk, and the LAST CTA of the grid to finish publishes completion —
// to the sender (its request's completion word) and, when the mailbox is device-visible, straight to the
// receiver (done[k] of the connection's mailbox), so the receiver's test() does not wait for the sender's proxy
// thread to notice.  Nothing stays resident between messages: a device-wide synchronisation of the application
// (cudaFree, cudaDeviceSynchronize) waits for at most the messages in flight, and a collective never depends on a
// kernel that has to be told to leave.
struct MsgArgs {
  const char* src;
  char* dst;
  uint64_t nbytes;      // bytes of SOURCE
  uint64_t chunk;       // source bytes per cluster (multiple of the op's unit)
  uint64_t* flag;       // sender-side completion word (pinned host memory)
  uint64_t flag_val;
  uint64_t* flag2;      // optional receiver-side completion word (mailbox, pinned host memory)
  uint64_t flag2_val;
  uint32_t* counter;    // device memory, zero on entry, reset to zero by the last CTA
  uint32_t op;
  float scale;
};
// Several messages in ONE launch: NCCL's proxy posts one isend per channel in a burst, and a launch per message costs the
// proxy thread ~6 us each (measured: 16 channels x 2 steps = ~190 us floor for every size up to 8 MiB).  The transport
// therefore collects the messages of a burst and launches them together: cluster c belongs to message i when
// first[i] <= c < first[i+1]; every message keeps its own completion counter and words.
constexpr int kMsgBatch = 16;
struct MsgBatch {
  int n;
  int group;                  // 0: CTAs are grouped by the hardware cluster; > 0: logical groups of that many consecutive CTAs
                              // in a plain launch (BNET_MSG_CLUSTER=0: no co-scheduling constraint on a busy GPU)
  int first[kMsgBatch + 1];   // first cluster of message i (prefix sums); first[n] = clusters in the grid
  MsgArgs m[kMsgBatch];
};
__global__ void __launch_bounds__(kThreads, 1) bnet_nvl_msg_kernel(const __grid_constant__ MsgBatch b) {
  const uint32_t csize = b.group > 0 ? (uint32_t)b.group : ptx::cluster_nctarank();
  const uint32_t crank = b.group > 0 ? blockIdx.x % csize : ptx::cluster_ctarank();
  const int cid = (int)(blockIdx.x / csize);
  int i = 0;
  while (i + 1 < b.n && cid >= b.first[i + 1]) i++;
  const MsgArgs& a = b.m[i];
  const uint32_t lc = (uint32_t)(cid - b.first[i]);                 // this cluster's chunk of message i
  const uint32_t nctas = (uint32_t)(b.first[i + 1] - b.first[i]) * csize;
  if (a.op != OP_FLUSH) {
    const size_t off = (size_t)lc * a.chunk;
    const size_t n = off >= a.nbytes ? 0 : (a.nbytes - off < a.chunk ? a.nbytes - off : a.chunk);
    size_t b0, b1;
    cta_share(a.op, n, crank, csize, &b0, &b1);
    process_range(a.op, a.src + off + b0, a.dst + dst_offset_for(a.op, off + b0), b1 - b0, threadIdx.x, kThreads, a.scale);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    ptx::fence_acq_rel_sys();                       // this CTA's (peer) stores before its arrival
    const uint32_t prev = atomicAdd(a.counter, 1u);
    if (prev == nctas - 1) {                        // every other CTA of this message has arrived (and fenced) before us
      *(volatile uint32_t*)a.counter = 0;           // ready for the next message that gets this counter
      ptx::fence_acq_rel_sys();
      if (a.flag2) ptx::st_release_sys_u64(a.flag2, a.flag2_val);
      ptx::st_release_sys_u64(a.flag, a.flag_val);
    }
  }
}

// ------------------------------------------------------------------ host side
namespace {

struct Stream {
  ClusterQ* q = nullptr;       // pinned host
  ClusterQ* q_dev = nullptr;   // device alias
  cudaStream_t stream = nullptr;
};

// Requests in flight on the NVL comms of this process (host-maintained, pinned, read by the kernels).
std::atomic<uint32_t>* g_outstanding_host = nullptr;
uint32_t* g_outstanding_dev = nullptr;
const uint32_t* outstanding_dev() {
  if (!g_outstanding_host) {
    void* dp = nullptr;
    void* hp = host_alloc_mapped(64, &dp);
    g_outstanding_host = new (hp) std::atomic<uint32_t>(0);
    g_outstanding_dev = (uint32_t*)dp;
  }
  return g_outstanding_dev;
}

// How a job reaches the GPU.  The transport (NCCL's isend) defaults to MODE_MSG: one launch per message and
// nothing resident; the extension API (P2PExecutor, benchmarks) defaults to the persistent cluster queues.
enum ExecMode : int { MODE_DEFAULT = -1, MODE_MSG = 0, MODE_PERSISTENT = 1, MODE_ONESHOT = 2, MODE_CE = 3 };
constexpr int kMsgCounters = 4096;   // completion counters of per-message launches (ring; far more than in flight)

struct Exec {
  int dev = -1;
  bool ok = false;
  bool persistent = true;
  int transport_mode = MODE_MSG;   // what exec_copy()/exec_flush() use (behind NCCL)
  int ext_mode = MODE_PERSISTENT;  // what bnet_exec_op() uses
  uint32_t* counters = nullptr;    // device memory, kMsgCounters words, all zero between messages
  uint64_t msg_seq = 0;
  MsgBatch batch{};                // messages collected since the last launch (transport path only)
  std::atomic<int> batch_n{0};     // == batch.n, readable without the lock (exec_kick's fast path)
  uint64_t batch_t0 = 0;
  uint64_t last_submit_ns = 0, burst_until_ns = 0;   // the batching window only applies while isends arrive back to back
  bool msg_cluster = true;     // BNET_MSG_CLUSTER=0: the per-message kernel is launched without a cluster dimension
  bool tma = false;
  bool ce = false;             // BNET_COPY_ENGINE=ce: DMA copy engines + stream memory ops, no kernels at all
  int nclusters = 4;
  int cluster_size = 2;
  size_t min_chunk = 1 << 20;
  uint64_t idle_ns = 1000000;
  uint64_t arm_ns = 50000000;
  size_t rr = 0;               // persists across messages
  std::vector<Stream> streams;
  std::mutex mu;
  ExecStats stats{};
  // single-grid mode (BNET_EXEC_GRID=1): all clusters in one kernel on one stream
  bool grid = false;
  GridCtl* ctl = nullptr;          // pinned host
  GridCtl* ctl_dev = nullptr;
  ClusterQ** queues = nullptr;     // pinned host array of the queues' device aliases
  ClusterQ** queues_dev = nullptr;
  cudaStream_t grid_stream = nullptr;
  uint64_t epoch = 0;
};

std::mutex g_mu;
Exec* g_exec[64] = {nullptr};

const char* mode_name(int m) {
  return m == MODE_MSG ? "per-message launch" : m == MODE_PERSISTENT ? "resident cluster kernels" : m == MODE_ONESHOT ? "launch per chunk"
         : m == MODE_CE ? "copy engines" : "default";
}

template <typename K>
cudaError_t launch_cluster(K kernel, int nblocks, int cluster, size_t smem, cudaStream_t st, void** args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(nblocks);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelExC(&cfg, (const void*)kernel, args);
}

Exec* get_exec(int dev) {
  if (dev < 0 || dev >= 64) return nullptr;
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_exec[dev]) return g_exec[dev]->ok ? g_exec[dev] : nullptr;
  CallScope cs_("executor setup");
  if (g_exec[dev]) return g_exec[dev]->ok ? g_exec[dev] : nullptr;
  Exec* e = new Exec();
  g_exec[dev] = e;
  e->dev = dev;
  const Config& cfg = Config::get();
  long long nc = env_int("NCLUSTERS", 8);
  e->nclusters = (int)(nc < 1 ? 1 : nc > kMaxChunksPerJob ? kMaxChunksPerJob : nc);
  long long cs = env_int("CLUSTER_SIZE", 4);
  e->cluster_size = (int)(cs < 1 ? 1 : cs > 8 ? 8 : cs);
  e->min_chunk = (size_t)env_int("DEV_MIN_CHUNKSIZE", (long long)(cfg.min_chunksize < 262144 ? cfg.min_chunksize : 262144));
  if (e->min_chunk < 16) e->min_chunk = 16;
  e->persistent = env_int("PERSISTENT", 1) != 0;
  e->msg_cluster = env_int("MSG_CLUSTER", 1) != 0;
  e->tma = env_str("COPY_ENGINE", "ldst") == "tma";
  e->ce = env_str("COPY_ENGINE", "ldst") == "ce" && driver().ok && driver().StreamWriteValue64 != nullptr;
  {
    // BNET_EXEC_MODE=msg|persistent|oneshot|ce picks the mode for BOTH users; the older knobs keep their meaning
    // (BNET_PERSISTENT=0 -> one launch per chunk, =1 -> resident cluster kernels, BNET_COPY_ENGINE=ce -> DMA engines)
    const std::string m = env_str("EXEC_MODE", "");
    const std::string pers = env_str("PERSISTENT", "");
    int forced = MODE_DEFAULT;
    if (m == "msg") forced = MODE_MSG;
    else if (m == "persistent") forced = MODE_PERSISTENT;
    else if (m == "oneshot") forced = MODE_ONESHOT;
    else if (m == "ce") forced = MODE_CE;
    else if (!m.empty()) BNET_WARN("unknown BNET_EXEC_MODE '%s' (msg, persistent, oneshot or ce)", m.c_str());
    if (forced == MODE_DEFAULT && e->ce) forced = MODE_CE;
    if (forced == MODE_DEFAULT && !pers.empty()) forced = e->persistent ? MODE_PERSISTENT : MODE_ONESHOT;
    if (forced == MODE_DEFAULT && env_int("EXEC_GRID", 0) != 0) forced = MODE_PERSISTENT;
    if (forced == MODE_CE && !(driver().ok && driver().StreamWriteValue64 != nullptr)) {
      BNET_WARN("copy-engine mode needs cuStreamWriteValue64; using per-message kernels");
      forced = MODE_MSG;
    }
    if (forced != MODE_DEFAULT) e->transport_mode = e->ext_mode = forced;
    e->ce = e->transport_mode == MODE_CE;
    e->persistent = e->transport_mode == MODE_PERSISTENT || e->ext_mode == MODE_PERSISTENT;
  }
  e->idle_ns = (uint64_t)env_int("KERNEL_IDLE_US", 1000) * 1000ull;
  e->arm_ns = (uint64_t)env_int("KERNEL_ARM_MS", 50) * 1000000ull;
  int cur = -1;
  cudaGetDevice(&cur);
  if (cur != dev) cudaSetDevice(dev);
  bool good = true;
  int lo = 0, hi = 0;
  cudaDeviceGetStreamPriorityRange(&lo, &hi);
  for (int i = 0; i < e->nclusters && good; i++) {
    Stream s;
    void* dp = nullptr;
    s.q = (ClusterQ*)host_alloc_mapped(sizeof(ClusterQ), &dp);
    s.q_dev = (ClusterQ*)dp;
    if (!s.q || cudaStreamCreateWithPriority(&s.stream, cudaStreamNonBlocking, hi) != cudaSuccess) good = false;
    e->streams.push_back(s);
  }
  if (good && e->tma) {
    cudaError_t err = cudaFuncSetAttribute(bnet_nvl_stream_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           kTmaStages * kTmaStageBytes);
    if (err != cudaSuccess) { cudaGetLastError(); e->tma = false; }
  }
  if (good) {
    // CUDA loads kernels lazily, and loading one may need to synchronise the context
    // (tools/blocking_calls_probe.py: a first launch waits for every running kernel).
    // On the data path that is a dead-lock: the NCCL kernel that is running is waiting for this
    // very transfer.  So load AND run every kernel once now, in the setup phase.
    cudaFuncAttributes fa;
    cudaFuncGetAttributes(&fa, bnet_nvl_stream_kernel<false>);
    cudaFuncGetAttributes(&fa, bnet_nvl_stream_kernel<true>);
    cudaFuncGetAttributes(&fa, bnet_nvl_oneshot_kernel);
    cudaFuncGetAttributes(&fa, bnet_nvl_msg_kernel);
    if (cudaMalloc((void**)&e->counters, kMsgCounters * sizeof(uint32_t)) != cudaSuccess ||
        cudaMemsetAsync(e->counters, 0, kMsgCounters * sizeof(uint32_t), e->streams[0].stream) != cudaSuccess) {
      cudaGetLastError();
      e->counters = nullptr;
      good = false;
    }
    void* wdp = nullptr;
    uint64_t* wflag = good ? (uint64_t*)host_alloc_mapped(64, &wdp) : nullptr;
    if (wflag) {
      OneShotArgs a{nullptr, nullptr, 0, (uint64_t*)wdp, 1, OP_FLUSH, 1.0f};
      void* args[] = {&a};
      cudaError_t err = launch_cluster(bnet_nvl_oneshot_kernel, e->cluster_size, e->cluster_size, 0, e->streams[0].stream, args);
      {
        // the per-message kernel: load it, run it once (two clusters, fence only) and check its completion protocol
        // (two messages, three clusters: the batch lookup, both counters and all four completion words)
        MsgBatch wb{};
        wb.n = 2;
        wb.group = e->msg_cluster ? 0 : e->cluster_size;
        wb.first[0] = 0; wb.first[1] = 2; wb.first[2] = 3;
        wb.m[0] = MsgArgs{nullptr, nullptr, 0, 64, (uint64_t*)wdp + 1, 7, (uint64_t*)wdp + 2, 9, e->counters, OP_FLUSH, 1.0f};
        wb.m[1] = MsgArgs{nullptr, nullptr, 0, 64, (uint64_t*)wdp + 3, 7, nullptr, 0, e->counters + 1, OP_FLUSH, 1.0f};
        void* margs[] = {&wb};
        cudaError_t e3 = launch_cluster(bnet_nvl_msg_kernel, 3 * e->cluster_size, e->msg_cluster ? e->cluster_size : 1, 0,
                                        e->streams[0].stream, margs);
        if (e3 == cudaSuccess) e3 = cudaStreamSynchronize(e->streams[0].stream);
        if (e3 != cudaSuccess || ((volatile uint64_t*)wflag)[1] != 7 || ((volatile uint64_t*)wflag)[2] != 9 ||
            ((volatile uint64_t*)wflag)[3] != 7) {
          if (err == cudaSuccess) err = e3 != cudaSuccess ? e3 : cudaErrorUnknown;
        }
      }
      for (Stream& s : e->streams) {
        if (!e->persistent) break;
        // persistent kernel: start it with stop already requested so it loads, runs and leaves
        __atomic_store_n(&s.q->stop, 1u, __ATOMIC_RELEASE);
        __atomic_store_n(&s.q->state, ST_RUNNING, __ATOMIC_RELEASE);
        ClusterQ* qd = s.q_dev;
        uint64_t idle = e->idle_ns, wd = 0;
        const uint32_t* outp = outstanding_dev();
        void* pargs[] = {&qd, &idle, &wd, &outp};
        cudaError_t e2 = e->tma ? launch_cluster(bnet_nvl_stream_kernel<true>, e->cluster_size, e->cluster_size,
                                                 kTmaStages * kTmaStageBytes, s.stream, pargs)
                                : launch_cluster(bnet_nvl_stream_kernel<false>, e->cluster_size, e->cluster_size, 0,
                                                 s.stream, pargs);
        if (e2 != cudaSuccess) err = e2;
        if (cudaStreamSynchronize(s.stream) != cudaSuccess) err = cudaErrorUnknown;
        __atomic_store_n(&s.q->stop, 0u, __ATOMIC_RELEASE);
        __atomic_store_n(&s.q->state, ST_EXITED, __ATOMIC_RELEASE);
      }
      if (err != cudaSuccess || *(volatile uint64_t*)wflag != 1) {
        cudaGetLastError();
        BNET_WARN("nvl executor: warm-up launch failed (%s)", cudaGetErrorString(err));
        good = false;
      }
      // (the 64-byte flag is deliberately not freed: cudaFreeHost waits for running kernels)
    }
  }
  if (good && e->persistent && env_int("EXEC_GRID", 0) != 0) {
    // single-grid mode: control block + the table of queue addresses, one stream, and the same
    // "load and run once with stop requested" warm-up as above
    void *cdp = nullptr, *qdp = nullptr;
    e->ctl = (GridCtl*)host_alloc_mapped(sizeof(GridCtl), &cdp);
    e->ctl_dev = (GridCtl*)cdp;
    e->queues = (ClusterQ**)host_alloc_mapped(sizeof(ClusterQ*) * kMaxChunksPerJob, &qdp);
    e->queues_dev = (ClusterQ**)qdp;
    bool ok = e->ctl && e->queues &&
              cudaStreamCreateWithPriority(&e->grid_stream, cudaStreamNonBlocking, hi) == cudaSuccess;
    if (ok && e->tma)
      ok = cudaFuncSetAttribute(bnet_nvl_grid_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                kTmaStages * kTmaStageBytes) == cudaSuccess;
    if (ok) {
      for (int i = 0; i < e->nclusters; i++) e->queues[i] = e->streams[i].q_dev;
      __atomic_store_n(&e->ctl->stop, 1u, __ATOMIC_RELEASE);
      __atomic_store_n(&e->ctl->state, ST_RUNNING, __ATOMIC_RELEASE);
      GridCtl* cd = e->ctl_dev;
      ClusterQ** qd = e->queues_dev;
      uint64_t ep = ++e->epoch, idle = e->idle_ns, wd = 0;
      const uint32_t* outp = outstanding_dev();
      void* gargs[] = {&cd, &qd, &ep, &idle, &wd, &outp};
      const int nblocks = e->nclusters * e->cluster_size;
      cudaError_t err = e->tma ? launch_cluster(bnet_nvl_grid_kernel<true>, nblocks, e->cluster_size,
                                                kTmaStages * kTmaStageBytes, e->grid_stream, gargs)
                               : launch_cluster(bnet_nvl_grid_kernel<false>, nblocks, e->cluster_size, 0, e->grid_stream, gargs);
      if (err != cudaSuccess || cudaStreamSynchronize(e->grid_stream) != cudaSuccess) ok = false;
      __atomic_store_n(&e->ctl->stop, 0u, __ATOMIC_RELEASE);
      __atomic_store_n(&e->ctl->state, ST_EXITED, __ATOMIC_RELEASE);
    }
    if (!ok) {
      cudaGetLastError();
      BNET_WARN("nvl executor: single-grid mode unavailable, using one kernel per cluster");
    }
    e->grid = ok;
  }
  if (cur != dev && cur >= 0) cudaSetDevice(cur);
  if (!good) cudaGetLastError();
  e->ok = good;
  BNET_INFO("nvl executor on dev %d: %d cluster(s) x %d CTA x %d thr, transport mode %s, engine=%s, min chunk %zu, idle %llu us",
            dev, e->nclusters, e->cluster_size, kThreads, e->grid ? "persistent single grid" : mode_name(e->transport_mode),
            e->ce ? "copy-engine" : e->tma ? "tma" : "ld/st", e->min_chunk, (unsigned long long)(e->idle_ns / 1000));
  return good ? e : nullptr;
}

int ensure_grid_running(Exec* e, bool arm) {
  for (int spin = 0;; spin++) {
    uint32_t st = __atomic_load_n(&e->ctl->state, __ATOMIC_ACQUIRE);
    if (st == ST_RUNNING) return 0;
    if (st == ST_EXITING) {   // cluster 0 is deciding; it settles on RUNNING or EXITED
      if (spin > 20000000) return -1;
      continue;
    }
    __atomic_store_n(&e->ctl->state, ST_RUNNING, __ATOMIC_RELEASE);
    GridCtl* cd = e->ctl_dev;
    ClusterQ** qd = e->queues_dev;
    uint64_t ep = ++e->epoch, idle = e->idle_ns, wd = arm ? e->arm_ns : 0;
    const uint32_t* outp = outstanding_dev();
    void* args[] = {&cd, &qd, &ep, &idle, &wd, &outp};
    const int nblocks = e->nclusters * e->cluster_size;
    cudaError_t err = e->tma ? launch_cluster(bnet_nvl_grid_kernel<true>, nblocks, e->cluster_size,
                                              kTmaStages * kTmaStageBytes, e->grid_stream, args)
                             : launch_cluster(bnet_nvl_grid_kernel<false>, nblocks, e->cluster_size, 0, e->grid_stream, args);
    if (err != cudaSuccess) {
      cudaGetLastError();
      __atomic_store_n(&e->ctl->state, ST_EXITED, __ATOMIC_RELEASE);
      BNET_WARN("nvl executor: grid launch failed: %s", cudaGetErrorString(err));
      return -1;
    }
    e->stats.launches++;
    return 0;
  }
}

int ensure_running(Exec* e, Stream& s, bool arm = false) {
  if (e->grid) return ensure_grid_running(e, arm);
  for (int spin = 0;; spin++) {
    uint32_t st = __atomic_load_n(&s.q->state, __ATOMIC_ACQUIRE);
    if (st == ST_RUNNING) return 0;
    if (st == ST_EXITING) {   // the kernel is deciding; it will settle on RUNNING or EXITED
      if (spin > 20000000) return -1;
      continue;
    }
    // EXITED: (re)launch
    __atomic_store_n(&s.q->state, ST_RUNNING, __ATOMIC_RELEASE);
    ClusterQ* qd = s.q_dev;
    uint64_t idle = e->idle_ns, wd = arm ? e->arm_ns : 0;
    const uint32_t* outp = outstanding_dev();
    void* args[] = {&qd, &idle, &wd, &outp};
    cudaError_t err = e->tma ? launch_cluster(bnet_nvl_stream_kernel<true>, e->cluster_size, e->cluster_size,
                                              kTmaStages * kTmaStageBytes, s.stream, args)
                             : launch_cluster(bnet_nvl_stream_kernel<false>, e->cluster_size, e->cluster_size, 0,
                                              s.stream, args);
    if (err != cudaSuccess) {
      cudaGetLastError();
      __atomic_store_n(&s.q->state, ST_EXITED, __ATOMIC_RELEASE);
      BNET_WARN("nvl executor: kernel launch failed: %s", cudaGetErrorString(err));
      return -1;
    }
    e->stats.launches++;
    return 0;
  }
}

// launches what MODE_MSG submissions have collected (e->mu held, e->dev current)
int flush_batch_locked(Exec* e) {
  MsgBatch& b = e->batch;
  if (b.n == 0) return 0;
  Stream& s = e->streams[e->rr];                    // the stream rotates per launch: successive bursts overlap on the device
  e->rr = (e->rr + 1) % e->streams.size();
  b.group = e->msg_cluster ? 0 : e->cluster_size;
  void* args[] = {&b};
  cudaError_t err;
  {
    CallScope cl_("cudaLaunchKernelEx(msg batch)");
    err = launch_cluster(bnet_nvl_msg_kernel, b.first[b.n] * e->cluster_size, e->msg_cluster ? e->cluster_size : 1, 0, s.stream, args);
  }
  e->stats.launches++;
  e->stats.batched += (uint64_t)b.n;
  b.n = 0;
  e->batch_n.store(0, std::memory_order_release);
  if (err != cudaSuccess) {
    cudaGetLastError();
    BNET_WARN("nvl executor: message launch failed: %s", cudaGetErrorString(err));
    return -1;
  }
  return 0;
}

int submit(Exec* e, int mode, uint32_t op, const void* src, void* dst, size_t nbytes, uint64_t* flags_dev, uint64_t flag_value,
           int* nchunks_out, float scale = 1.0f, uint64_t* flag2_dev = nullptr, uint64_t flag2_value = 0, int defer_launch = 0) {
  CallScope cs_("exec submit");
  std::lock_guard<std::mutex> lk(e->mu);
  int cur = -1;
  cudaGetDevice(&cur);
  if (cur != e->dev) cudaSetDevice(e->dev);
  if (mode == MODE_DEFAULT) mode = e->ext_mode;
  if (mode == MODE_CE && op != OP_COPY) mode = MODE_MSG;            // fused ops need SMs
  if (mode == MODE_PERSISTENT && !e->persistent) mode = MODE_MSG;   // resident kernels were not set up
  size_t unit = src_unit_for(op) < 64 ? 64 : src_unit_for(op);   // keep chunk cuts vector aligned on both sides
  // (copy-engine mode pays two driver calls per chunk: only split what is large enough to keep several engines busy)
  const size_t min_chunk = (mode == MODE_CE && e->min_chunk < ((size_t)2 << 20)) ? ((size_t)2 << 20) : e->min_chunk;
  size_t cs = chunk_size(nbytes, min_chunk, (size_t)e->nclusters);
  cs = (cs + unit - 1) / unit * unit;
  int nchunks = nbytes ? (int)((nbytes + cs - 1) / cs) : 1;
  if (nchunks > kMaxChunksPerJob) nchunks = kMaxChunksPerJob;   // cannot happen: nclusters <= kMaxChunksPerJob
  int rc = 0;
  if (mode == MODE_MSG) {
    // The message joins the pending batch; the batch is launched when it is full, when the caller asked for an immediate
    // launch (extension API), or by exec_kick() — which the transport calls from test(), i.e. right after NCCL's proxy has
    // posted the isends of one pass over its channels.  One launch then carries all of them.
    MsgArgs a{(const char*)src, (char*)dst, nbytes, cs, flags_dev, flag_value, flag2_dev, flag2_value,
              e->counters + (e->msg_seq++ % kMsgCounters), op, scale};
    MsgBatch& b = e->batch;
    {
      // two isends within 3 us of each other = NCCL's proxy is walking its channels: batch for the next 2 ms.  A lone
      // message (small collectives on one channel) is launched at once, so the window costs it nothing.
      const uint64_t t = now_ns();
      if (t - e->last_submit_ns < 3000) e->burst_until_ns = t + 2000000;
      e->last_submit_ns = t;
      if (b.n == 0) { b.first[0] = 0; e->batch_t0 = t; }
    }
    b.m[b.n] = a;
    b.first[b.n + 1] = b.first[b.n] + nchunks;
    b.n++;
    e->batch_n.store(b.n, std::memory_order_release);
    if (defer_launch == 0 || b.n == kMsgBatch || now_ns() >= e->burst_until_ns) rc = flush_batch_locked(e);
    e->stats.chunks += nchunks;
    e->stats.jobs++;
    e->stats.bytes += nbytes;
    if (cur != e->dev && cur >= 0) cudaSetDevice(cur);
    *nchunks_out = 1;   // one completion word per message
    return rc;
  }
  for (int c = 0; c < nchunks && rc == 0; c++) {
    size_t off = (size_t)c * cs;
    size_t n = nbytes ? (nbytes - off < cs ? nbytes - off : cs) : 0;
    Stream& s = e->streams[e->rr];
    e->rr = (e->rr + 1) % e->streams.size();
    if (mode == MODE_CE) {
      // copy-engine mode: a DMA copy, then a stream-ordered 64-bit write of the completion word.  No SM is
      // used and nothing stays resident between messages; the price is two driver calls per chunk.
      // (driver-level unified-address copy: the destination is a VMM / IPC mapping of the peer's memory)
      cudaError_t err = cudaSuccess;
      if (n) {
        if (driver().MemcpyAsync)
          err = driver().MemcpyAsync((CUdeviceptr)((char*)dst + off), (CUdeviceptr)((const char*)src + off), n, (CUstream)s.stream) == CUDA_SUCCESS
                    ? cudaSuccess : cudaErrorUnknown;
        else
          err = cudaMemcpyAsync((char*)dst + off, (const char*)src + off, n, cudaMemcpyDefault, s.stream);
      }
      if (err != cudaSuccess ||
          driver().StreamWriteValue64((CUstream)s.stream, (CUdeviceptr)(flags_dev + c), flag_value, 0) != CUDA_SUCCESS) {
        cudaGetLastError();
        rc = -1;
      }
      e->stats.launches++;
      e->stats.chunks++;
      continue;
    }
    if (mode == MODE_PERSISTENT) {
      uint64_t t = s.q->tail;
      uint64_t spins = 0;
      while (t - __atomic_load_n(&s.q->head, __ATOMIC_ACQUIRE) >= (uint64_t)kQueueDepth) {
        if (ensure_running(e, s) != 0 || ++spins > 200000000ull) { rc = -1; break; }
      }
      if (rc) break;
      Desc& d = s.q->d[t % kQueueDepth];
      d.src = (const char*)src + off;
      d.dst = (char*)dst + dst_offset_for(op, off);
      d.nbytes = n;
      d.flag = flags_dev + c;
      d.flag_val = flag_value;
      d.op = op;
      d.scale = scale;
      __atomic_store_n(&d.seq, t + 1, __ATOMIC_RELEASE);
      s.q->tail = t + 1;
      if (e->grid) __atomic_store_n(&e->ctl->submitted, e->ctl->submitted + 1, __ATOMIC_RELEASE);
      __atomic_thread_fence(__ATOMIC_SEQ_CST);   // publish, then look at the kernel's state (Dekker)
      rc = ensure_running(e, s);
      e->stats.persistent++;
    } else {
      OneShotArgs a{(const char*)src + off, (char*)dst + dst_offset_for(op, off), n, flags_dev + c, flag_value, op, scale};
      void* args[] = {&a};
      cudaError_t err = launch_cluster(bnet_nvl_oneshot_kernel, e->cluster_size, e->cluster_size, 0, s.stream, args);
      if (err != cudaSuccess) {
        cudaGetLastError();
        rc = -1;
      }
      e->stats.launches++;
    }
    e->stats.chunks++;
  }
  e->stats.jobs++;
  e->stats.bytes += nbytes;
  if (cur != e->dev && cur >= 0) cudaSetDevice(cur);
  *nchunks_out = nchunks;
  return rc;
}

}  // namespace

// One message of the transport: OP_COPY for NCCL's isend, any other ExecOp for the fused-collective extension
// (bnet_isend_op): the receiver's buffer is accumulated into / converted on the way instead of overwritten.
int exec_transfer(int dev, uint32_t op, float scale, const void* src, void* dst, size_t nbytes, volatile uint64_t* flags_host,
                  uint64_t* flags_dev, uint64_t flag_value, int* nchunks, uint64_t* flag2_dev, uint64_t flag2_value) {
  if (fake()) {   // CPU emulation: the kernels' own per-CTA body run by one "thread", same completion protocol
    if (op == OP_COPY) memcpy(dst, src, nbytes);
    else process_range(op, (const char*)src, (char*)dst, nbytes, 0, 1, scale);
    size_t cs = chunk_size(nbytes, (size_t)env_int("DEV_MIN_CHUNKSIZE", 262144), 4);
    int n = nbytes ? (int)((nbytes + cs - 1) / cs) : 1;
    if (op != OP_COPY) n = 1;
    for (int i = 0; i < n; i++) flags_host[i] = flag_value;
    *nchunks = n;
    return 0;
  }
  Exec* e = get_exec(dev);
  if (!e) return -1;
  static const int batching = (int)env_int("MSG_BATCH", 1);     // BNET_MSG_BATCH=0: one launch per message, immediately
  return submit(e, e->transport_mode, op, src, dst, nbytes, flags_dev, flag_value, nchunks, scale, flag2_dev, flag2_value, batching);
}

// Launch whatever the transport has queued for `dev` (called from test(): cheap when nothing is pending).
void exec_kick(int dev) {
  if (dev < 0 || dev >= 64) return;
  Exec* e = g_exec[dev];
  if (!e || !e->ok || e->batch_n.load(std::memory_order_acquire) == 0) return;
  // NCCL tests a request right after posting it, so "launch at the next test()" alone would never see more than one
  // message: give the burst a few microseconds to arrive (the proxy posts its channels back to back), then launch.
  static const uint64_t window_ns = (uint64_t)env_int("MSG_BATCH_US", 4) * 1000ull;
  std::lock_guard<std::mutex> lk(e->mu);
  if (e->batch.n == 0) return;
  if (e->batch.n < kMsgBatch && now_ns() - e->batch_t0 < window_ns && now_ns() < e->burst_until_ns) return;
  int cur = -1;
  cudaGetDevice(&cur);
  if (cur != e->dev) cudaSetDevice(e->dev);
  flush_batch_locked(e);
  if (cur != e->dev && cur >= 0) cudaSetDevice(cur);
}

size_t exec_dst_bytes(uint32_t op, size_t src_bytes) { return dst_offset_for(op, src_bytes); }

int exec_copy(int dev, const void* src, void* dst, size_t nbytes, volatile uint64_t* flags_host, uint64_t* flags_dev,
              uint64_t flag_value, int* nchunks, uint64_t* flag2_dev, uint64_t flag2_value) {
  return exec_transfer(dev, OP_COPY, 1.0f, src, dst, nbytes, flags_host, flags_dev, flag_value, nchunks, flag2_dev, flag2_value);
}

int exec_flush(int dev, volatile uint64_t* flag_host, uint64_t* flag_dev, uint64_t flag_value) {
  if (fake()) {
    *flag_host = flag_value;
    return 0;
  }
  Exec* e = get_exec(dev);
  if (!e) return -1;
  int n = 0;
  return submit(e, e->transport_mode == MODE_CE ? MODE_MSG : e->transport_mode, OP_FLUSH, nullptr, nullptr, 0, flag_dev, flag_value, &n);
}

// Extension entry point: fused move+reduce / move+cast between registered buffers
// (used by tests, bench/p2p_bw and the Python ops layer).
extern "C" __attribute__((visibility("default"))) int bnet_exec_op(int dev, uint32_t op, const void* src, void* dst, size_t src_bytes,
                            volatile uint64_t* flags_host, uint64_t* flags_dev, uint64_t flag_value, int* nchunks) {
  if (fake()) return exec_copy(dev, src, dst, src_bytes, flags_host, flags_dev, flag_value, nchunks);
  Exec* e = get_exec(dev);
  if (!e) return -1;
  return submit(e, MODE_DEFAULT, op, src, dst, src_bytes, flags_dev, flag_value, nchunks);
}

extern "C" __attribute__((visibility("default"))) int bnet_exec_op_scaled(int dev, uint32_t op, const void* src, void* dst, size_t src_bytes,
                                   uint64_t* flags_dev, uint64_t flag_value, float scale, int* nchunks) {
  Exec* e = get_exec(dev);
  if (!e) return -1;
  return submit(e, MODE_DEFAULT, op, src, dst, src_bytes, flags_dev, flag_value, nchunks, scale);
}

int exec_op_mode(int dev, int mode, uint32_t op, const void* src, void* dst, size_t src_bytes, uint64_t* flags_dev,
                 uint64_t flag_value, float scale, int* nchunks) {
  Exec* e = get_exec(dev);
  if (!e) return -1;
  return submit(e, mode, op, src, dst, src_bytes, flags_dev, flag_value, nchunks, scale);
}
extern "C" __attribute__((visibility("default"))) int bnet_exec_op_mode(int dev, int mode, uint32_t op, const void* src, void* dst,
                                 size_t src_bytes, uint64_t* flags_dev, uint64_t flag_value, float scale, int* nchunks) {
  return exec_op_mode(dev, mode, op, src, dst, src_bytes, flags_dev, flag_value, scale, nchunks);
}

void exec_outstanding_add(int delta) {
  if (g_outstanding_host) g_outstanding_host->fetch_add((uint32_t)delta, std::memory_order_relaxed);
}

int exec_prepare(int dev) {
  if (fake()) return 0;
  Exec* e = get_exec(dev);
  if (!e) return -1;
  if (e->transport_mode != MODE_PERSISTENT || e->arm_ns == 0) return 0;   // only the resident-kernel mode has anything to arm
  // Arm: have the stream kernels resident BEFORE the first message so that the data path
  // needs no kernel launch (one that could be held up by a device-synchronising call
  // elsewhere in the process while the NCCL kernel it serves is already waiting).
  std::lock_guard<std::mutex> lk(e->mu);
  int cur = -1;
  cudaGetDevice(&cur);
  if (cur != e->dev) cudaSetDevice(e->dev);
  int rc = 0;
  if (e->grid) {
    rc = ensure_grid_running(e, /*arm=*/true);
  } else {
    for (Stream& s : e->streams)
      if (ensure_running(e, s, /*arm=*/true) != 0) rc = -1;
  }
  if (cur != e->dev && cur >= 0) cudaSetDevice(cur);
  return rc;
}

void exec_dump() {
  static const char* names[] = {"EXITED", "RUNNING", "EXITING"};
  std::lock_guard<std::mutex> lk(g_mu);
  for (Exec* e : g_exec) {
    if (!e || !e->ok) continue;
    fprintf(stderr, "[bnet watchdog] executor dev %d: %s%s%s, %d x %d CTAs, outstanding %u, jobs %llu chunks %llu launches %llu\n",
            e->dev, e->grid ? "single grid" : mode_name(e->transport_mode), e->tma ? " tma" : "", e->ce ? " copy-engine" : "",
            e->nclusters, e->cluster_size, g_outstanding_host ? g_outstanding_host->load() : 0u,
            (unsigned long long)e->stats.jobs, (unsigned long long)e->stats.chunks, (unsigned long long)e->stats.launches);
    if (e->grid && e->ctl)
      fprintf(stderr, "[bnet watchdog]   grid state %s stop %u submitted %llu epoch %llu\n", names[e->ctl->state % 3], e->ctl->stop,
              (unsigned long long)e->ctl->submitted, (unsigned long long)e->epoch);
    for (size_t i = 0; i < e->streams.size(); i++) {
      ClusterQ* q = e->streams[i].q;
      if (!q) continue;
      fprintf(stderr, "[bnet watchdog]   queue %zu: kernel %s stop %u published %llu completed %llu%s\n", i, names[q->state % 3], q->stop,
              (unsigned long long)q->tail, (unsigned long long)q->head,
              cudaStreamQuery(e->streams[i].stream) == cudaSuccess ? " (stream idle)" : " (stream busy)");
    }
  }
}

void exec_stats(ExecStats* out) {
  memset(out, 0, sizeof(*out));
  std::lock_guard<std::mutex> lk(g_mu);
  for (Exec* e : g_exec) {
    if (!e) continue;
    out->jobs += e->stats.jobs;
    out->chunks += e->stats.chunks;
    out->bytes += e->stats.bytes;
    out->launches += e->stats.launches;
    out->persistent += e->stats.persistent;
    out->batched += e->stats.batched;
  }
}

void exec_shutdown() {
  std::lock_guard<std::mutex> lk(g_mu);
  for (Exec* e : g_exec) {
    if (!e || !e->ok) continue;
    for (Stream& s : e->streams)
      if (s.q) __atomic_store_n(&s.q->stop, 1u, __ATOMIC_RELEASE);
    if (e->ctl) __atomic_store_n(&e->ctl->stop, 1u, __ATOMIC_RELEASE);
  }
}

}  // namespace cuda
}  // namespace bnet

// Device copy executor used by the NVLink transport: moves a registered buffer
// into the peer GPU's buffer with sm_90a kernels (K1/K8 in SURVEY.md §2.6).
//
// A transfer is split into chunks of max(ceil(n/nclusters), MIN_CHUNKSIZE) bytes —
// the same rule the reference uses to stripe a message over its TCP streams
// (reference: src/utils.rs:200-205, nthread_…:405-413) — and the chunks are dealt
// round-robin to thread-block clusters ("device streams"), the cursor persisting
// across messages.  Every chunk has its own completion word in pinned host memory
// that the kernel writes with release.sys semantics after its stores; test()
// polls those words: no syscall, no mutex on the completion path.
#pragma once
#include <cstddef>
#include <cstdint>

namespace bnet {
namespace cuda {

constexpr int kMaxChunksPerJob = 16;

struct ExecStats {
  uint64_t jobs, chunks, bytes, launches, persistent;
  uint64_t batched;      // messages that left in a multi-message launch (per-message mode)
};

// flags_host/flags_dev: the same kMaxChunksPerJob words seen from host and device.
// On return *nchunks words will eventually hold `flag_value`.
// Returns 0 on success, <0 on failure (caller falls back to the bounce ring).
// flag2_dev (optional): a second completion word the kernel publishes BEFORE the first — the receiver-visible
// done[k] of the connection's mailbox — honoured by the per-message mode; callers must not rely on it.
int exec_copy(int dev, const void* src, void* dst, size_t nbytes, volatile uint64_t* flags_host,
              uint64_t* flags_dev, uint64_t flag_value, int* nchunks, uint64_t* flag2_dev = nullptr,
              uint64_t flag2_value = 0);
// the general form: `op` is an ExecOp of csrc/cuda/exec_body.cuh (0 = copy); nbytes counts SOURCE bytes
int exec_transfer(int dev, uint32_t op, float scale, const void* src, void* dst, size_t nbytes, volatile uint64_t* flags_host,
                  uint64_t* flags_dev, uint64_t flag_value, int* nchunks, uint64_t* flag2_dev = nullptr, uint64_t flag2_value = 0);
// per-message mode collects the isends of a burst; this launches them (the transport calls it from test())
void exec_kick(int dev);
// destination bytes an op writes for `src_bytes` of input (casts change the size)
size_t exec_dst_bytes(uint32_t op, size_t src_bytes);
// extension entry point with an explicit mode (-1 default, 0 per-message launch, 1 resident queues, 2 launch per chunk, 3 copy engines)
int exec_op_mode(int dev, int mode, uint32_t op, const void* src, void* dst, size_t src_bytes, uint64_t* flags_dev,
                 uint64_t flag_value, float scale, int* nchunks);
// Device-side fence used by iflush (K7): completes `flag` once prior peer stores are visible.
int exec_flush(int dev, volatile uint64_t* flag_host, uint64_t* flag_dev, uint64_t flag_value);
// Create streams / queues / pinned memory for `dev` now (setup phase) instead of at the first job.
int exec_prepare(int dev);
// +1 when a request is posted on an NVL comm, -1 when it completes: the stream kernels stay resident
// while the count is non-zero so that no kernel launch is needed in the middle of a collective.
void exec_outstanding_add(int delta);
void exec_stats(ExecStats* out);
// Watchdog helper: one line per executor queue (kernel state, published/completed descriptors) to stderr.
void exec_dump();
void exec_shutdown();

}  // namespace cuda
}  // namespace bnet

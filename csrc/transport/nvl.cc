// NVL transport: intra-host connections that never touch a socket on the data
// path.  This is the new capability the reference does not have (it is TCP-only,
// host pointers only: reference nthread_…:252, cc/v4/nccl_net_v4.cc:105-109).
//
// Rendezvous: connect() dials the listener's abstract unix socket, creates a
// POSIX shm "mailbox" and names it in the hello; accept() maps it.  No reply is
// needed, so connect never waits for the peer's accept (NCCL proxy friendly).
//
// Mailbox protocol, message k of a connection (strict FIFO like the reference,
// SURVEY.md §2.2 "Protocol invariant"):
//   receiver irecv : rdesc[k%S] = {capacity, mr, offset, type}; seq=k+1 (release)
//   sender   isend : waits for rdesc seq, then announces ann[k%S] = {nbytes, path}
//     direct path  : dst is a registered CUDA buffer we could import ->
//                    sm_90a copy kernel writes the peer buffer over NVLink, one
//                    completion word per chunk; host then publishes done[k%S]
//     ring path    : payload streams through an SPSC byte ring in the shm
//                    (host<->host, or CUDA staged with private-stream copies)
//   both           : test() polls memory only — no syscalls, no locks shared with
//                    other comms (the reference takes a global mutex per call,
//                    src/lib.rs:15)
// regMr(NCCL_PTR_CUDA) on the receiver exports the allocation (CUDA IPC handle
// or cuMem POSIX fd passed with SCM_RIGHTS) into the mailbox's MR table; the
// sender imports lazily on first use.
#include <errno.h>
#include <fcntl.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/socket.h>
#include <sys/stat.h>
#include <sys/prctl.h>
#include <sys/uio.h>
#include <sys/un.h>
#include <unistd.h>

#include <deque>
#include <map>
#include <mutex>
#include <thread>
#include <vector>

#include "core/engine.h"
#include "core/telemetry.h"
#include "cuda/cuda_iface.h"
#include "cuda/nvl_exec.h"

namespace bnet {
namespace {

constexpr int kSlots = kMaxRequests;
constexpr int kMaxMr = 128;
constexpr uint32_t kNoMr = 0xffffffffu;
constexpr uint32_t kShmMagic = 0x4e564c31u;  // "NVL1"
constexpr size_t kRingBudget = 1 << 20;      // bytes copied per progress() call
constexpr size_t kCmaBudget = 4 << 20;       // bytes pulled per progress() call and request (single-copy path)

struct alignas(64) RecvDesc {
  std::atomic<uint64_t> seq;
  uint64_t capacity;
  uint64_t offset;      // dst address - allocation base (valid when mr_idx != kNoMr)
  uint32_t mr_idx;
  uint32_t dst_type;
  int32_t tag;
};
enum : uint32_t { PATH_DIRECT = 0, PATH_RING = 1, PATH_CMA = 2 };
struct alignas(64) Announce {
  std::atomic<uint64_t> seq;
  uint64_t nbytes;
  uint32_t via_ring;      // PATH_*
  int32_t err;
  uint64_t src_addr;      // PATH_CMA: where the payload sits in the sender's address space
};
struct alignas(64) Done {
  std::atomic<uint64_t> seq;
  int32_t err;            // PATH_CMA: the receiver could not pull the payload
};
struct alignas(64) MrDesc {
  std::atomic<uint32_t> gen;      // odd = valid
  uint32_t type;
  uint64_t addr, size;
  cuda::MemExport exp;
};

struct NvlShm {
  uint32_t magic, version;
  uint64_t total_bytes, ring_bytes;
  alignas(64) std::atomic<uint32_t> sender_closed;
  alignas(64) std::atomic<uint32_t> receiver_closed;
  alignas(64) std::atomic<uint64_t> ring_w;
  alignas(64) std::atomic<uint64_t> ring_r;
  // cross-memory attach (single copy for large host messages): the receiver pulls straight from the sender's
  // buffer with process_vm_readv.  Probed once at accept: 0 = not probed yet, 1 = works, 2 = refused by the kernel
  alignas(64) std::atomic<uint32_t> cma_state;
  uint64_t cma_probe_addr, cma_probe_val;
  RecvDesc rdesc[kSlots];
  Announce ann[kSlots];
  Done done[kSlots];
  MrDesc mrs[kMaxMr];
  alignas(4096) char ring[1];
};

struct NvlHello {
  uint32_t magic;
  uint16_t version;
  uint16_t flags;
  uint64_t listen_nonce;
  uint32_t pid;
  int32_t cuda_dev;
  uint64_t shm_bytes;
  char shm_name[64];
};

enum NvlMsgType : uint32_t { MSG_MR_FD = 1 };
struct NvlMsg {
  uint32_t type;
  uint32_t mr_idx;
  uint32_t gen;
  uint32_t pad;
};

int send_fd(int sock, const NvlMsg& m, int fd) {
  msghdr mh{};
  iovec iov{const_cast<NvlMsg*>(&m), sizeof(m)};
  mh.msg_iov = &iov;
  mh.msg_iovlen = 1;
  char cbuf[CMSG_SPACE(sizeof(int))];
  memset(cbuf, 0, sizeof(cbuf));
  if (fd >= 0) {
    mh.msg_control = cbuf;
    mh.msg_controllen = sizeof(cbuf);
    cmsghdr* c = CMSG_FIRSTHDR(&mh);
    c->cmsg_level = SOL_SOCKET;
    c->cmsg_type = SCM_RIGHTS;
    c->cmsg_len = CMSG_LEN(sizeof(int));
    memcpy(CMSG_DATA(c), &fd, sizeof(int));
  }
  for (;;) {
    ssize_t n = sendmsg(sock, &mh, MSG_NOSIGNAL);
    if (n == (ssize_t)sizeof(m)) return kOk;
    if (n < 0 && (errno == EINTR)) continue;
    if (n < 0 && (errno == EAGAIN || errno == EWOULDBLOCK)) { usleep(50); continue; }
    return kErrSystem;
  }
}

// 1 = got a message, 0 = nothing pending, <0 = peer gone
int recv_fd(int sock, NvlMsg* m, int* fd) {
  msghdr mh{};
  iovec iov{m, sizeof(*m)};
  mh.msg_iov = &iov;
  mh.msg_iovlen = 1;
  char cbuf[CMSG_SPACE(sizeof(int))];
  mh.msg_control = cbuf;
  mh.msg_controllen = sizeof(cbuf);
  *fd = -1;
  ssize_t n = recvmsg(sock, &mh, MSG_DONTWAIT | MSG_CMSG_CLOEXEC);
  if (n == 0) return -1;
  if (n < 0) return (errno == EAGAIN || errno == EWOULDBLOCK || errno == EINTR) ? 0 : -1;
  if (n != (ssize_t)sizeof(*m)) return -1;
  for (cmsghdr* c = CMSG_FIRSTHDR(&mh); c; c = CMSG_NXTHDR(&mh, c))
    if (c->cmsg_level == SOL_SOCKET && c->cmsg_type == SCM_RIGHTS) memcpy(fd, CMSG_DATA(c), sizeof(int));
  return 1;
}

class NvlComm;
void watchdog_register(NvlComm* c);
void watchdog_unregister(NvlComm* c);

class NvlComm : public Comm {
 public:
  NvlComm(Kind k, int dev_, int uds, NvlShm* shm, size_t shm_bytes, std::string shm_name, uint32_t peer_pid,
          int peer_dev)
      : Comm(k), uds_(uds), shm_(shm), shm_bytes_(shm_bytes), shm_name_(std::move(shm_name)), peer_pid_(peer_pid),
        peer_dev_(peer_dev) {
    dev = dev_;
    ring_bytes_ = shm->ring_bytes;
    local_dev_ = cuda::current_device();
    if (cuda::available()) {
      void* dp = nullptr;
      shm_registered_ = cuda::host_register(shm_, shm_bytes_, &dp) == 0;
      if (shm_registered_) shm_dev_ = (char*)dp;
      if (k == SEND) {
        void* fdp = nullptr;
        flags_ = (uint64_t*)cuda::host_alloc_mapped(sizeof(uint64_t) * kSlots * cuda::kMaxChunksPerJob, &fdp);
        flags_dev_ = (uint64_t*)fdp;
      }
    }
    set_nonblocking(uds_, true);
    cma_min_ = (size_t)env_int("CMA_MIN", 512 << 10);   // below this the ring (cache-resident, pipelined) is as fast
    if (k == RECV) {
      // can we read the sender's memory directly?  (same uid + ptrace permission; the sender opted in with
      // PR_SET_PTRACER_ANY for hosts that run the Yama LSM)
      uint32_t verdict = 2;
      if (env_int("CMA", 1) != 0 && shm_->cma_probe_addr) {
        uint64_t val = 0;
        iovec l{&val, sizeof(val)}, r{(void*)shm_->cma_probe_addr, sizeof(val)};
        if (process_vm_readv((pid_t)peer_pid_, &l, 1, &r, 1, 0) == (ssize_t)sizeof(val) && val == shm_->cma_probe_val) verdict = 1;
      }
      shm_->cma_state.store(verdict, std::memory_order_release);
      BNET_DEBUG("nvl accept: cross-memory attach to pid %u %s", peer_pid_, verdict == 1 ? "works" : "unavailable");
    }
    // all CUDA resource creation happens here, in NCCL's setup phase, never on the data path
    cuda_live_ = cuda::available() && !cuda::fake();
    if (cuda_live_) cuda::exec_prepare(local_dev_);
    watchdog_register(this);
  }

  ~NvlComm() override {
    watchdog_unregister(this);
    (kind == SEND ? shm_->sender_closed : shm_->receiver_closed).store(1, std::memory_order_release);
    for (auto& kv : imports_)
      if (kv.second.base) cuda::release_import(kv.second.exp, kv.second.base, kv.second.cookie);
    for (auto& im : stale_) cuda::release_import(im.exp, im.base, im.cookie);
    for (auto& kv : fds_) close(kv.second);
    for (auto& kv : exports_) cuda::release_export(&kv.second);
    if (flags_) cuda::host_free_mapped(flags_);
    if (shm_registered_) cuda::host_unregister(shm_);
    munmap(shm_, shm_bytes_);
    if (kind == SEND) shm_unlink(shm_name_.c_str());   // creator unlinks; mappings stay valid
    close(uds_);
  }

  const char* transport() const override { return "nvl"; }

  // ---- memory registration --------------------------------------------------------
  int reg_mr(void* data, size_t size, int type, MemHandle** out) override {
    if (type != NCCL_PTR_HOST && type != NCCL_PTR_CUDA) return kErrInvalid;
    if (type == NCCL_PTR_CUDA && !cuda::available()) return kErrInvalid;
    std::lock_guard<std::mutex> lk(mu_);
    MemHandle* mh = new MemHandle;
    mh->addr = data;
    mh->size = size;
    mh->type = type;
    mh->owner = this;
    mh->id = kNoMr;
    if (kind == RECV && type == NCCL_PTR_CUDA) {
      // publish the allocation so the sender's kernels can store into it directly
      int idx = -1;
      for (int i = 0; i < kMaxMr; i++)
        if ((shm_->mrs[i].gen.load(std::memory_order_relaxed) & 1) == 0) { idx = i; break; }
      cuda::MemExport exp;
      if (idx >= 0 && cuda::export_memory(data, size, &exp) == 0) {
        MrDesc& d = shm_->mrs[idx];
        uint32_t gen = d.gen.load(std::memory_order_relaxed) + 1;  // becomes odd
        d.type = (uint32_t)type;
        d.addr = (uint64_t)data;
        d.size = size;
        d.exp = exp;
        bool ok = true;
        if (exp.kind == cuda::EXPORT_POSIX_FD && exp.pid != peer_pid_) {
          NvlMsg m{MSG_MR_FD, (uint32_t)idx, gen, 0};
          ok = send_fd(uds_, m, exp.fd) == kOk;
        }
        if (ok) {
          d.gen.store(gen, std::memory_order_release);
          exports_[idx] = exp;
          mh->id = (uint32_t)idx;
          BNET_DEBUG("nvl regMr: %p +%zu exported as mr %d (kind %u)", data, size, idx, exp.kind);
        } else {
          cuda::release_export(&exp);
        }
      } else {
        BNET_INFO("nvl regMr: %p +%zu not exportable; this buffer will use the bounce ring", data, size);
      }
    }
    if (kind == SEND && type == NCCL_PTR_HOST && size) {
      // Is this buffer readable through cross-memory attach?  Ordinary pages are; driver-owned mappings (pinned
      // CUDA host allocations are VM_PFNMAP on some stacks) are not.  Reading our own first and last byte with
      // the same system call takes the same get_user_pages path the receiver will take.
      char probe[2];
      iovec l[2] = {{&probe[0], 1}, {&probe[1], 1}};
      iovec rm[2] = {{data, 1}, {(char*)data + size - 1, 1}};
      mh->cma = process_vm_readv(getpid(), l, 2, rm, 2, 0) == 2 ? 1 : 0;
    }
    if (kind == SEND && type == NCCL_PTR_HOST && cuda::available()) {
      // BNET_HOST_SRC_DIRECT=1: pinned host sources (NCCL keeps its LL send buffers in host memory) are read by
      // the copy kernel itself and stored straight into the peer GPU, instead of ring + staged H2D copy
      static const bool host_direct = env_int("HOST_SRC_DIRECT", 0) != 0;
      if (host_direct) mh->priv = cuda::host_device_alias(data);
    }
    *out = mh;
    return kOk;
  }

  int dereg_mr(MemHandle* mh) override {
    std::lock_guard<std::mutex> lk(mu_);
    if (kind == RECV && mh->id != kNoMr) {
      MrDesc& d = shm_->mrs[mh->id];
      d.gen.fetch_add(1, std::memory_order_release);  // even = free; sender drops its import lazily
      auto it = exports_.find((int)mh->id);
      if (it != exports_.end()) {
        cuda::release_export(&it->second);
        exports_.erase(it);
      }
    }
    delete mh;
    return kOk;
  }

  // ---- posting ------------------------------------------------------------------------
  int isend(const void* data, size_t size, int tag, MemHandle* mh, Request** out) override {
    return isend_op(data, size, tag, mh, 0 /* OP_COPY */, 1.0f, out);
  }

  // op != 0: the sender's kernel accumulates into / converts into the receiver's posted buffer (K4 / K5 fused with the move)
  int isend_op(const void* data, size_t size, int tag, MemHandle* mh, uint32_t op, float scale, Request** out) override {
    *out = nullptr;
    if (kind != SEND) return kErrInvalid;
    if (op != 0 && !(mh && mh->type == NCCL_PTR_CUDA)) return kErrInvalid;   // fused ops exist on the device path only
    std::lock_guard<std::mutex> lk(mu_);
    int b = broken.load(std::memory_order_acquire);
    if (b) return b;
    Request* r = alloc_req(REQ_SEND, const_cast<void*>(data), size, tag, mh);
    if (!r) return kOk;
    track(+1);
    r->u[0] = seq_++;   // message index
    r->u[1] = 0;        // stage
    r->u[4] = op;
    memcpy(&r->u[5], &scale, sizeof(scale));
    pending_.push_back(r);
    progress_locked();
    *out = r;
    return kOk;
  }

  int irecv(void* data, size_t size, int tag, MemHandle* mh, Request** out) override {
    *out = nullptr;
    if (kind != RECV) return kErrInvalid;
    std::lock_guard<std::mutex> lk(mu_);
    int b = broken.load(std::memory_order_acquire);
    if (b) return b;
    Request* r = alloc_req(REQ_RECV, data, size, tag, mh);
    if (!r) return kOk;
    // the first receive of a burst is the earliest sign of a collective on this GPU: make sure this
    // process' stream kernels are resident before its own isends need them
    if (track(+1) == 0 && cuda_live_) cuda::exec_prepare(local_dev_);
    uint64_t k = seq_++;
    r->u[0] = k;
    r->u[1] = 0;
    RecvDesc& d = shm_->rdesc[k % kSlots];
    d.capacity = size;
    d.tag = tag;
    d.dst_type = mh ? (uint32_t)mh->type : (uint32_t)NCCL_PTR_HOST;
    d.mr_idx = kNoMr;
    d.offset = 0;
    if (mh && mh->type == NCCL_PTR_CUDA && mh->id != kNoMr) {
      const MrDesc& m = shm_->mrs[mh->id];
      d.mr_idx = mh->id;
      d.offset = (uint64_t)data - m.exp.alloc_base;
    }
    d.seq.store(k + 1, std::memory_order_release);
    pending_.push_back(r);
    *out = r;
    return kOk;
  }

  int iflush(void* data, size_t size, MemHandle* mh, Request** out) override {
    // Data was stored by the peer's kernel and fenced at system scope before the
    // completion word became visible, so there is nothing left to flush; with
    // BNET_FLUSH_KERNEL=1 a device-side fence kernel (K7) is issued anyway.
    Request* r = alloc_req(REQ_FLUSH, data, size, 0, mh);
    if (!r) { *out = nullptr; return kOk; }
    static const bool use_kernel = env_int("FLUSH_KERNEL", 0) != 0;
    bool issued = false;
    if (use_kernel && flush_flags_ready() && mh && mh->type == NCCL_PTR_CUDA) {
      uint64_t v = ++flush_seq_;
      r->u[2] = v;
      r->u[3] = 1;
      issued = cuda::exec_flush(local_dev_, flush_flag_, flush_flag_dev_, v) == 0;
    }
    if (!issued) {
      r->u[3] = 0;
      r->ndone.store(1, std::memory_order_release);
    }
    *out = r;
    return kOk;
  }

  int test(Request* r, int* done, size_t* size) override {
    if (cuda_live_) cuda::exec_kick(local_dev_);   // launch the isends of this burst (one kernel for all of them)
    {
      std::lock_guard<std::mutex> lk(mu_);
      if (r->kind == REQ_FLUSH && r->u[3] == 1 && !r->complete() &&
          *(volatile uint64_t*)flush_flag_ >= r->u[2])
        r->ndone.store(1, std::memory_order_release);
      progress_locked();
    }
    return Comm::test(r, done, size);
  }

  void progress() override {}   // test() drives progress under the comm lock

  // BNET_WATCHDOG_MS: describe a comm whose oldest request is older than the threshold
  bool dump_if_stuck(uint64_t older_than_ns) {
    std::unique_lock<std::mutex> lk(mu_, std::try_to_lock);
    if (!lk.owns_lock() || pending_.empty()) return false;
    Request* r = pending_.front();
    uint64_t age = now_ns() - r->t_post;
    if (age < older_than_ns) return false;
    uint64_t k = r->u[0];
    const RecvDesc& d = shm_->rdesc[k % kSlots];
    fprintf(stderr,
            "[bnet watchdog] %s comm %llu pid %d dev %d peer pid %u: %zu pending, head msg %llu stage %llu size %zu "
            "moved %llu age %.1f ms | rdesc.seq %llu cap %llu mr %u type %u | ann.seq %llu nbytes %llu ring %u err %d | "
            "done.seq %llu | ring w %llu r %llu | next seq %llu\n",
            kind == SEND ? "send" : "recv", (unsigned long long)id, (int)getpid(), local_dev_, peer_pid_, pending_.size(),
            (unsigned long long)k, (unsigned long long)r->u[1], r->size, (unsigned long long)r->u[2], age / 1e6,
            (unsigned long long)d.seq.load(), (unsigned long long)d.capacity, d.mr_idx, d.dst_type,
            (unsigned long long)shm_->ann[k % kSlots].seq.load(), (unsigned long long)shm_->ann[k % kSlots].nbytes,
            shm_->ann[k % kSlots].via_ring, shm_->ann[k % kSlots].err, (unsigned long long)shm_->done[k % kSlots].seq.load(),
            (unsigned long long)shm_->ring_w.load(), (unsigned long long)shm_->ring_r.load(), (unsigned long long)seq_);
    if (kind == SEND && r->u[1] == 2 && flags_) {
      volatile uint64_t* fh = flags_ + (k % kSlots) * cuda::kMaxChunksPerJob;
      fprintf(stderr, "[bnet watchdog]   chunk flags (%llu expected %llu):", (unsigned long long)r->u[2], (unsigned long long)(k + 1));
      for (uint64_t c = 0; c < r->u[2]; c++) fprintf(stderr, " %llu", (unsigned long long)fh[c]);
      fprintf(stderr, "\n");
    }
    return true;
  }

 private:
  bool flush_flags_ready() {
    if (flush_flag_) return true;
    if (!cuda::available()) return false;
    void* dp = nullptr;
    flush_flag_ = (uint64_t*)cuda::host_alloc_mapped(64, &dp);
    flush_flag_dev_ = (uint64_t*)dp;
    return flush_flag_ != nullptr;
  }

  void fail_pending(int st) {
    broken.store(st, std::memory_order_release);
    for (Request* r : pending_) {
      r->fail(st);
      r->ndone.store(r->nsub.load(), std::memory_order_release);
      track(-1);
    }
    pending_.clear();
  }

  bool peer_alive() {
    if ((kind == SEND ? shm_->receiver_closed : shm_->sender_closed).load(std::memory_order_acquire)) return false;
    uint64_t now = now_ns();
    if (now - last_alive_check_ < 20000000ull) return true;  // 20 ms
    last_alive_check_ = now;
    if (kind == SEND) {
      drain_uds();
      return !uds_eof_;
    }
    char c;
    ssize_t n = recv(uds_, &c, 1, MSG_DONTWAIT | MSG_PEEK);
    return !(n == 0 || (n < 0 && errno != EAGAIN && errno != EWOULDBLOCK && errno != EINTR));
  }

  void drain_uds() {
    for (;;) {
      NvlMsg m;
      int fd;
      int r = recv_fd(uds_, &m, &fd);
      if (r == 0) return;
      if (r < 0) { uds_eof_ = true; return; }
      if (m.type == MSG_MR_FD && fd >= 0) {
        auto it = fds_.find(m.mr_idx);
        if (it != fds_.end()) close(it->second);
        fds_[m.mr_idx] = fd;
        fd_gen_[m.mr_idx] = m.gen;
      } else if (fd >= 0) {
        close(fd);
      }
    }
  }

  struct Import {
    uint32_t gen = 0;
    void* base = nullptr;
    void* cookie = nullptr;
    bool failed = false;
    cuda::MemExport exp;
  };

  // returns the local address of (mr, offset) or nullptr (retry=true: not yet importable)
  char* resolve(uint32_t mr_idx, uint64_t offset, bool* retry) {
    *retry = false;
    if (mr_idx >= (uint32_t)kMaxMr) return nullptr;
    MrDesc& d = shm_->mrs[mr_idx];
    uint32_t gen = d.gen.load(std::memory_order_acquire);
    if (!(gen & 1)) return nullptr;
    Import& im = imports_[mr_idx];
    if (im.gen != gen) {
      // unmapping waits for running kernels (tools/blocking_calls_probe.py): never on the data path
      if (im.base) stale_.push_back(im);
      im = Import();
      im.gen = gen;
      im.exp = d.exp;
      int fd = -1;
      if (d.exp.kind == cuda::EXPORT_POSIX_FD && d.exp.pid != (uint64_t)getpid()) {
        drain_uds();
        auto it = fds_.find(mr_idx);
        if (it == fds_.end() || fd_gen_[mr_idx] != gen) {
          im.gen = 0;   // fd still in flight on the unix socket
          *retry = true;
          return nullptr;
        }
        fd = it->second;
      }
      if (cuda::import_memory(d.exp, fd, local_dev_, &im.base, &im.cookie) != 0) {
        im.failed = true;
        im.base = nullptr;
        BNET_INFO("nvl: could not import peer mr %u; falling back to the bounce ring", mr_idx);
      }
      if (fd >= 0) {
        close(fd);
        fds_.erase(mr_idx);
      }
    }
    if (im.failed || !im.base) return nullptr;
    return (char*)im.base + offset;
  }

  size_t ring_write(const char* src, size_t n, bool src_cuda) {
    uint64_t w = shm_->ring_w.load(std::memory_order_relaxed);
    uint64_t rd = shm_->ring_r.load(std::memory_order_acquire);
    size_t freeb = ring_bytes_ - (size_t)(w - rd);
    if (n > freeb) n = freeb;
    size_t done = 0;
    while (done < n) {
      size_t pos = (size_t)((w + done) % ring_bytes_);
      size_t seg = ring_bytes_ - pos < n - done ? ring_bytes_ - pos : n - done;
      if (src_cuda) {
        if (cuda::memcpy_sync(shm_->ring + pos, src + done, seg, local_dev_) != 0) return (size_t)-1;
      } else {
        memcpy(shm_->ring + pos, src + done, seg);
      }
      done += seg;
    }
    shm_->ring_w.store(w + n, std::memory_order_release);
    return n;
  }

  size_t ring_read(char* dst, size_t n, bool dst_cuda) {
    uint64_t rd = shm_->ring_r.load(std::memory_order_relaxed);
    uint64_t w = shm_->ring_w.load(std::memory_order_acquire);
    size_t avail = (size_t)(w - rd);
    if (n > avail) n = avail;
    size_t done = 0;
    while (done < n) {
      size_t pos = (size_t)((rd + done) % ring_bytes_);
      size_t seg = ring_bytes_ - pos < n - done ? ring_bytes_ - pos : n - done;
      if (dst_cuda) {
        if (cuda::memcpy_sync(dst + done, shm_->ring + pos, seg, local_dev_) != 0) return (size_t)-1;
      } else {
        memcpy(dst + done, shm_->ring + pos, seg);
      }
      done += seg;
    }
    shm_->ring_r.store(rd + n, std::memory_order_release);
    return n;
  }

  // requests in flight across all NVL comms of the process (see cuda::exec_outstanding_add)
  static int track(int delta) {
    static std::atomic<int> n{0};
    int before = n.fetch_add(delta);
    cuda::exec_outstanding_add(delta);
    return before;
  }

  void complete(Request* r, size_t nbytes) {
    track(-1);
    r->nbytes.store(nbytes, std::memory_order_relaxed);
    r->ndone.store(r->nsub.load(std::memory_order_relaxed), std::memory_order_release);
  }

  void progress_locked() {
    if (pending_.empty()) return;
    if (kind == SEND) progress_send(); else progress_recv();
    if (!pending_.empty() && !peer_alive()) {
      // The peer is gone, but what it already announced / wrote into the mailbox is still
      // valid (a sender may legitimately close right after its last isend completed):
      // drain until nothing moves any more, then fail whatever is left.
      for (;;) {
        uint64_t before = moved_;
        size_t npend = pending_.size();
        if (kind == SEND) progress_send(); else progress_recv();
        if (pending_.empty() || (moved_ == before && pending_.size() == npend)) break;
      }
      if (!pending_.empty()) {
        BNET_WARN("nvl: peer (pid %u) went away with %zu request(s) in flight", peer_pid_, pending_.size());
        fail_pending(kErrRemote);
      }
    }
  }

  // stages: 0 = waiting for the receiver's descriptor, 1 = streaming through the ring,
  //         2 = direct copy in flight, 3 = finished (to be removed)
  void progress_send() {
    Telemetry& T = Telemetry::get();
    bool ring_busy = false;   // ring payloads are strictly serial
    size_t budget = kRingBudget;
    for (Request* r : pending_) {
      uint64_t k = r->u[0];
      if (r->u[1] == 0) {
        if (ring_busy) break;  // keep announce order == ring order simple: one ring writer at a time
        RecvDesc& d = shm_->rdesc[k % kSlots];
        if (d.seq.load(std::memory_order_acquire) != k + 1) break;  // FIFO: later messages wait too
        Announce& a = shm_->ann[k % kSlots];
        const uint32_t op = (uint32_t)r->u[4];
        const size_t dst_bytes = op ? cuda::exec_dst_bytes(op, r->size) : r->size;
        if (dst_bytes > d.capacity) {
          BNET_WARN("nvl isend: %zu bytes do not fit the posted receive (%llu)", dst_bytes, (unsigned long long)d.capacity);
          a.nbytes = dst_bytes;
          a.via_ring = 0;
          a.err = kErrInvalid;
          a.seq.store(k + 1, std::memory_order_release);
          r->fail(kErrInvalid);
          track(-1);
          r->u[1] = 3;
          continue;
        }
        bool src_cuda = r->mh && r->mh->type == NCCL_PTR_CUDA;
        // what the copy kernel reads: the device buffer, or the device alias of a pinned host buffer
        const char* ksrc = src_cuda ? (const char*)r->buf : nullptr;
        if (!src_cuda && r->mh && r->mh->priv)
          ksrc = (const char*)r->mh->priv + ((const char*)r->buf - (const char*)r->mh->addr);
        char* dst = nullptr;
        if (r->size && ksrc && d.dst_type == NCCL_PTR_CUDA && d.mr_idx != kNoMr && flags_) {
          bool retry = false;
          dst = resolve(d.mr_idx, d.offset, &retry);
          if (retry) break;
        }
        int nchunks = 0;
        bool direct = false;
        if (dst) {
          uint64_t* fh = flags_ + (k % kSlots) * cuda::kMaxChunksPerJob;
          uint64_t* fd = flags_dev_ + (k % kSlots) * cuda::kMaxChunksPerJob;
          // the kernel itself publishes done[k] to the receiver when it can see the mailbox (one proxy hop less);
          // the host repeats the store when it notices completion, which also covers the other executor modes
          uint64_t* done_dev = shm_dev_ ? (uint64_t*)(shm_dev_ + ((char*)&shm_->done[k % kSlots].seq - (char*)shm_)) : nullptr;
          float scale = 1.0f;
          memcpy(&scale, &r->u[5], sizeof(scale));
          direct = cuda::exec_transfer(local_dev_, op, scale, ksrc, dst, r->size, fh, fd, k + 1, &nchunks, done_dev, k + 1) == 0;
        }
        if (op != 0 && !direct) {
          // a fused op cannot fall back to the byte paths: tell the receiver, fail the request
          BNET_WARN("nvl isend_op: op %u needs registered CUDA buffers on both sides (direct path unavailable)", op);
          a.nbytes = dst_bytes;
          a.via_ring = 0;
          a.err = kErrInvalid;
          a.seq.store(k + 1, std::memory_order_release);
          r->fail(kErrInvalid);
          track(-1);
          r->u[1] = 3;
          continue;
        }
        // large host -> host message: let the receiver pull it straight out of our buffer (one copy, none by us)
        const bool cma = !direct && !src_cuda && d.dst_type == NCCL_PTR_HOST && r->size >= cma_min_ && r->mh &&
                         r->mh->cma == 1 && shm_->cma_state.load(std::memory_order_acquire) == 1;
        a.nbytes = dst_bytes;
        a.via_ring = direct ? PATH_DIRECT : cma ? PATH_CMA : PATH_RING;
        r->prof_path = direct ? 3 : cma ? 2 : 1;   // BNET_PROF_PATH_* (include/bnet/bnet_profiler.h)
        a.src_addr = (uint64_t)r->buf;
        a.err = 0;
        a.seq.store(k + 1, std::memory_order_release);
        if (cma) {
          r->u[1] = 4;
          T.m().cma_msgs.fetch_add(1, std::memory_order_relaxed);
        } else if (direct) {
          r->u[1] = 2;
          r->u[2] = (uint64_t)nchunks;
          T.m().nvl_kernel_chunks.fetch_add((uint64_t)nchunks, std::memory_order_relaxed);
        } else if (r->size == 0) {
          complete(r, 0);
          r->u[1] = 3;
          continue;
        } else {
          r->u[1] = 1;
          r->u[2] = 0;  // bytes written
        }
      }
      if (r->u[1] == 1) {
        if (ring_busy) continue;
        bool src_cuda = r->mh && r->mh->type == NCCL_PTR_CUDA;
        size_t left = r->size - (size_t)r->u[2];
        size_t want = left < budget ? left : budget;
        size_t n = want ? ring_write((const char*)r->buf + r->u[2], want, src_cuda) : 0;
        if (n == (size_t)-1) {
          r->fail(kErrCuda);
          track(-1);
          r->u[1] = 3;
          broken.store(kErrCuda);
          continue;
        }
        r->u[2] += n;
        budget -= n;
        moved_ += n;
        T.m().shm_bytes_total.fetch_add(n, std::memory_order_relaxed);
        if (r->u[2] == r->size) {
          T.on_chunk_sent(r->size, now_ns() - r->t_post);
          complete(r, r->size);
          r->u[1] = 3;
        } else {
          ring_busy = true;
        }
      } else if (r->u[1] == 4) {
        Done& dn = shm_->done[k % kSlots];
        if (dn.seq.load(std::memory_order_acquire) == k + 1) {
          if (dn.err) {
            r->fail(dn.err);
            track(-1);
            broken.store(dn.err);
          } else {
            moved_ += r->size;
            T.on_chunk_sent(r->size, now_ns() - r->t_post);
            complete(r, r->size);
          }
          r->u[1] = 3;
        }
      } else if (r->u[1] == 2) {
        volatile uint64_t* fh = flags_ + (k % kSlots) * cuda::kMaxChunksPerJob;
        bool all = true;
        for (uint64_t c = 0; c < r->u[2]; c++)
          if (fh[c] != k + 1) { all = false; break; }
        if (all) {
          std::atomic_thread_fence(std::memory_order_acquire);
          shm_->done[k % kSlots].seq.store(k + 1, std::memory_order_release);
          T.m().nvl_bytes_total.fetch_add(r->size, std::memory_order_relaxed);
          T.on_chunk_sent(r->size, now_ns() - r->t_post);
          complete(r, r->size);
          r->u[1] = 3;
        }
      }
    }
    while (!pending_.empty() && pending_.front()->u[1] == 3) pending_.pop_front();
    // requests finished out of order stay in the deque until the head finishes; drop them now
    for (auto it = pending_.begin(); it != pending_.end();)
      if ((*it)->u[1] == 3) it = pending_.erase(it); else ++it;
  }

  void progress_recv() {
    Telemetry& T = Telemetry::get();
    size_t budget = kRingBudget;
    bool ring_busy = false;
    for (Request* r : pending_) {
      uint64_t k = r->u[0];
      Announce& a = shm_->ann[k % kSlots];
      if (r->u[1] == 0) {
        if (a.seq.load(std::memory_order_acquire) != k + 1) break;  // sender announces in order
        if (a.err) {
          r->fail(a.err);
          track(-1);
          r->u[1] = 3;
          continue;
        }
        r->u[4] = a.nbytes;
        r->prof_path = a.via_ring == PATH_RING ? 1 : a.via_ring == PATH_CMA ? 2 : 3;
        r->u[1] = a.via_ring == PATH_RING ? 1 : a.via_ring == PATH_CMA ? 4 : 2;
        r->u[2] = 0;
        r->u[5] = a.src_addr;
        if (a.via_ring == PATH_RING && a.nbytes == 0) {
          complete(r, 0);
          r->u[1] = 3;
          continue;
        }
      }
      if (r->u[1] == 1) {
        if (ring_busy) continue;
        bool dst_cuda = r->mh && r->mh->type == NCCL_PTR_CUDA;
        size_t left = (size_t)(r->u[4] - r->u[2]);
        size_t want = left < budget ? left : budget;
        size_t n = want ? ring_read((char*)r->buf + r->u[2], want, dst_cuda) : 0;
        if (n == (size_t)-1) {
          r->fail(kErrCuda);
          track(-1);
          r->u[1] = 3;
          broken.store(kErrCuda);
          continue;
        }
        r->u[2] += n;
        budget -= n;
        moved_ += n;
        if (r->u[2] == r->u[4]) {
          T.on_chunk_recv((uint64_t)r->u[4]);
          complete(r, (size_t)r->u[4]);
          r->u[1] = 3;
        } else {
          ring_busy = true;   // the ring is a byte stream: later ring messages wait for this one
        }
      } else if (r->u[1] == 4) {
        // pull a bounded piece per call so that one huge message cannot monopolise the proxy thread
        size_t left = (size_t)(r->u[4] - r->u[2]);
        size_t want = left < kCmaBudget ? left : kCmaBudget;
        iovec l{(char*)r->buf + r->u[2], want}, rm{(void*)(r->u[5] + r->u[2]), want};
        ssize_t n = want ? process_vm_readv((pid_t)peer_pid_, &l, 1, &rm, 1, 0) : 0;
        Done& dn = shm_->done[k % kSlots];
        if (n < 0) {
          BNET_WARN("nvl: process_vm_readv from pid %u failed: %s", peer_pid_, strerror(errno));
          dn.err = kErrSystem;
          dn.seq.store(k + 1, std::memory_order_release);
          r->fail(kErrSystem);
          track(-1);
          r->u[1] = 3;
          broken.store(kErrSystem);
          continue;
        }
        r->u[2] += (uint64_t)n;
        moved_ += (uint64_t)n;
        if (r->u[2] == r->u[4]) {
          dn.err = 0;
          dn.seq.store(k + 1, std::memory_order_release);   // the sender may reuse its buffer now
          T.m().shm_bytes_total.fetch_add(r->u[4], std::memory_order_relaxed);
          T.on_chunk_recv((uint64_t)r->u[4]);
          complete(r, (size_t)r->u[4]);
          r->u[1] = 3;
        }
      } else if (r->u[1] == 2) {
        if (shm_->done[k % kSlots].seq.load(std::memory_order_acquire) == k + 1) {
          T.on_chunk_recv((uint64_t)r->u[4]);
          complete(r, (size_t)r->u[4]);
          r->u[1] = 3;
        }
      }
    }
    for (auto it = pending_.begin(); it != pending_.end();)
      if ((*it)->u[1] == 3) it = pending_.erase(it); else ++it;
  }

  int uds_;
  NvlShm* shm_;
  size_t shm_bytes_, ring_bytes_ = 0;
  std::string shm_name_;
  uint32_t peer_pid_;
  int peer_dev_, local_dev_ = -1;
  bool shm_registered_ = false, uds_eof_ = false, cuda_live_ = false;
  char* shm_dev_ = nullptr;     // device alias of the mailbox (kernels publish done[k] straight to the receiver)
  std::mutex mu_;
  std::deque<Request*> pending_;
  uint64_t seq_ = 0;
  uint64_t last_alive_check_ = 0;
  uint64_t moved_ = 0;          // bytes moved through the ring (progress detector)
  uint64_t* flags_ = nullptr;
  uint64_t* flags_dev_ = nullptr;
  uint64_t* flush_flag_ = nullptr;
  uint64_t* flush_flag_dev_ = nullptr;
  uint64_t flush_seq_ = 0;
  size_t cma_min_ = 512 << 10;
  std::map<uint32_t, Import> imports_;
  std::vector<Import> stale_;
  std::map<uint32_t, int> fds_;
  std::map<uint32_t, uint32_t> fd_gen_;
  std::map<int, cuda::MemExport> exports_;
};

std::mutex g_wd_mu;
std::vector<NvlComm*> g_wd_comms;
bool g_wd_started = false;

// BNET_WATCHDOG_MS (default 20000, 0 = off): a request older than this gets its connection's state printed to
// stderr, together with every thread that has been inside a plugin call for that long and the executor's state.
// It only describes; failing a stuck request is BNET_TIMEOUT_MS's job.
void watchdog_register(NvlComm* c) {
  static const long long ms = env_int("WATCHDOG_MS", 20000);
  if (ms <= 0) return;
  std::lock_guard<std::mutex> lk(g_wd_mu);
  g_wd_comms.push_back(c);
  if (!g_wd_started) {
    g_wd_started = true;
    std::thread([] {
      const uint64_t thr = (uint64_t)ms * 1000000ull;
      for (int dumps = 0; dumps < 12;) {
        usleep((useconds_t)(thr / 2000));
        bool stuck = false;
        {
          std::lock_guard<std::mutex> lk(g_wd_mu);
          for (NvlComm* c : g_wd_comms) stuck |= c->dump_if_stuck(thr);
        }
        if (calltrace_dump(thr) > 0) stuck = true;
        if (stuck) {
          if (cuda::available() && !cuda::fake()) cuda::exec_dump();
          dumps++;
          usleep((useconds_t)(thr / 1000));   // one report per period is enough
        }
      }
    }).detach();
  }
}

void watchdog_unregister(NvlComm* c) {
  std::lock_guard<std::mutex> lk(g_wd_mu);
  for (size_t i = 0; i < g_wd_comms.size(); i++)
    if (g_wd_comms[i] == c) { g_wd_comms.erase(g_wd_comms.begin() + i); break; }
}

size_t shm_total(size_t ring) { return offsetof(NvlShm, ring) + ring; }

}  // namespace

bool nvl_available() { return true; }   // shared-memory path needs no GPU; CUDA paths are probed per buffer
size_t nvl_hello_size() { return sizeof(NvlHello); }

std::string nvl_uds_name(uint32_t pid, uint64_t listen_nonce) {
  char b[64];
  snprintf(b, sizeof(b), "bnet-%u-%016llx", pid, (unsigned long long)listen_nonce);
  return b;
}

Comm* nvl_connect(int dev, const Handle& h) {
  const Config& cfg = Config::get();
  int fd = socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
  if (fd < 0) return nullptr;
  sockaddr_un un{};
  un.sun_family = AF_UNIX;
  std::string name = nvl_uds_name(h.pid, h.listen_nonce);
  memcpy(un.sun_path + 1, name.data(), name.size());
  socklen_t ulen = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + name.size());
  if (::connect(fd, (sockaddr*)&un, ulen) != 0) {
    BNET_DEBUG("nvl connect: unix socket %s unreachable: %s", name.c_str(), strerror(errno));
    close(fd);
    return nullptr;
  }
  // mailbox
  size_t ring = cfg.shm_ring_bytes < 65536 ? 65536 : cfg.shm_ring_bytes;
  size_t total = shm_total(ring);
  char shm_name[64];
  snprintf(shm_name, sizeof(shm_name), "/bnet-%d-%016llx", (int)getpid(), (unsigned long long)random_u64());
  int sfd = shm_open(shm_name, O_CREAT | O_EXCL | O_RDWR, 0600);
  // posix_fallocate reserves the pages now: on a small /dev/shm we fall back to TCP here instead of
  // dying with SIGBUS at the first touch of an unbacked page (8 ranks x dozens of connections add up)
  if (sfd < 0 || ftruncate(sfd, (off_t)total) != 0 || posix_fallocate(sfd, 0, (off_t)total) != 0) {
    BNET_INFO("nvl connect: shm_open/ftruncate/fallocate(%zu) failed: %s", total, strerror(errno));
    if (sfd >= 0) { close(sfd); shm_unlink(shm_name); }
    close(fd);
    return nullptr;
  }
  void* p = mmap(nullptr, total, PROT_READ | PROT_WRITE, MAP_SHARED, sfd, 0);
  close(sfd);
  if (p == MAP_FAILED) {
    shm_unlink(shm_name);
    close(fd);
    return nullptr;
  }
  NvlShm* shm = (NvlShm*)p;   // fresh shm is zero-filled: all seq/gen counters start at 0
  shm->magic = kShmMagic;
  shm->version = kWireVersion;
  shm->total_bytes = total;
  shm->ring_bytes = ring;
  {
    // let the receiver verify (and later use) cross-memory attach on us
    static uint64_t probe_word = 0;
    static std::once_flag once;
    std::call_once(once, [] {
      probe_word = random_u64() | 1;
#ifdef PR_SET_PTRACER
      prctl(PR_SET_PTRACER, PR_SET_PTRACER_ANY, 0, 0, 0);   // Yama: allow same-uid peers to read our memory
#endif
    });
    shm->cma_probe_addr = (uint64_t)&probe_word;
    shm->cma_probe_val = probe_word;
  }
  std::atomic_thread_fence(std::memory_order_release);
  NvlHello hello{};
  hello.magic = kHandleMagic;
  hello.version = kWireVersion;
  hello.listen_nonce = h.listen_nonce;
  hello.pid = (uint32_t)getpid();
  hello.cuda_dev = cuda::current_device();
  hello.shm_bytes = total;
  snprintf(hello.shm_name, sizeof(hello.shm_name), "%s", shm_name);
  if (write_all(fd, &hello, sizeof(hello), nullptr, 5000) != kOk) {
    munmap(p, total);
    shm_unlink(shm_name);
    close(fd);
    return nullptr;
  }
  BNET_DEBUG("nvl connect: mailbox %s (%zu bytes) to pid %u", shm_name, total, h.pid);
  return new NvlComm(Comm::SEND, dev, fd, shm, total, shm_name, h.pid, h.cuda_dev);
}

Comm* nvl_accept(int dev, int uds_fd, const void* hello_buf, size_t hello_len) {
  if (hello_len != sizeof(NvlHello)) return nullptr;
  NvlHello hello;
  memcpy(&hello, hello_buf, sizeof(hello));
  hello.shm_name[sizeof(hello.shm_name) - 1] = 0;
  if (hello.magic != kHandleMagic || hello.version != kWireVersion) {
    BNET_WARN("nvl accept: bad hello (magic %x version %u)", hello.magic, hello.version);
    return nullptr;
  }
  int sfd = shm_open(hello.shm_name, O_RDWR, 0600);
  if (sfd < 0) {
    BNET_WARN("nvl accept: cannot open mailbox %s: %s", hello.shm_name, strerror(errno));
    return nullptr;
  }
  void* p = mmap(nullptr, hello.shm_bytes, PROT_READ | PROT_WRITE, MAP_SHARED, sfd, 0);
  close(sfd);
  if (p == MAP_FAILED) return nullptr;
  NvlShm* shm = (NvlShm*)p;
  if (shm->magic != kShmMagic || shm->total_bytes != hello.shm_bytes) {
    munmap(p, hello.shm_bytes);
    return nullptr;
  }
  shm_unlink(hello.shm_name);   // both ends hold a mapping now; nothing leaks if a process dies
  return new NvlComm(Comm::RECV, dev, uds_fd, shm, hello.shm_bytes, hello.shm_name, hello.pid, hello.cuda_dev);
}

}  // namespace bnet

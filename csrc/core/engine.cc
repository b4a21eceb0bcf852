#include "core/engine.h"

#include <dlfcn.h>
#include <errno.h>
#include <poll.h>
#include <string.h>
#include <sys/un.h>
#include <unistd.h>

#include <nvtx3/nvToolsExt.h>

#include "bnet/bnet_profiler.h"
#include "core/telemetry.h"
#include "cuda/cuda_iface.h"
#include "cuda/nvl_exec.h"

namespace bnet {

// ------------------------------------------------------------------ NCCL profiler hook (ncclNet v10)
static std::atomic<ncclProfilerCallback_t> g_prof_fn{nullptr};

void profiler_set_callback(ncclProfilerCallback_t fn) { g_prof_fn.store(fn, std::memory_order_release); }

static void prof_fill(const Request* r, bnetProfilerEventDescr_v1_t* d, bool stop) {
  memset(d, 0, sizeof(*d));
  d->type = r->kind == REQ_SEND ? BNET_PROF_ISEND : BNET_PROF_IRECV;
  d->path = stop ? r->prof_path : 0;
  d->tag = r->tag;
  d->comm_id = r->comm ? r->comm->id : 0;
  d->request_id = r->id;
  d->length = stop ? (size_t)r->nbytes.load(std::memory_order_relaxed) : r->size;
}

void profiler_start(Request* r, void* parent_handle) {
  ncclProfilerCallback_t fn = g_prof_fn.load(std::memory_order_acquire);
  if (!fn || !parent_handle || !r || r->kind == REQ_FLUSH) return;
  bnetProfilerEventDescr_v1_t d;
  prof_fill(r, &d, false);
  void* eh = nullptr;
  if (fn(&eh, 0 /* start */, parent_handle, BNET_PROFILER_PLUGIN_ID, &d) == ncclSuccess) r->prof_event = eh;
}

void profiler_stop(Request* r) {
  ncclProfilerCallback_t fn = g_prof_fn.load(std::memory_order_acquire);
  if (!fn || !r->prof_event) return;
  bnetProfilerEventDescr_v1_t d;
  prof_fill(r, &d, true);
  void* eh = r->prof_event;
  r->prof_event = nullptr;
  fn(&eh, 1 /* stop */, nullptr, BNET_PROFILER_PLUGIN_ID, &d);
}

// ------------------------------------------------------------------ Comm base
static std::atomic<uint64_t> g_comm_ids{1};

// BNET_NVTX=1: one NVTX range per request (isend/irecv -> completion), visible in Nsight Systems
// next to NCCL's own ranges — the on-box replacement for the reference's Jaeger spans.
static bool nvtx_on() {
  static const bool on = env_int("NVTX", 0) != 0;
  return on;
}

Comm::Comm(Kind k) : kind(k) { id = g_comm_ids.fetch_add(1); }
Comm::~Comm() {}

int Comm::reg_mr(void* data, size_t size, int type, MemHandle** out) {
  // Host memory needs no registration for sockets.  The reference accepts only
  // NCCL_PTR_HOST and never writes *mhandle (cc/v4/nccl_net_v4.cc:105-109).
  if (type != NCCL_PTR_HOST) return kErrInvalid;
  MemHandle* mh = new MemHandle;
  mh->addr = data;
  mh->size = size;
  mh->type = type;
  mh->id = next_mr.fetch_add(1);
  mh->owner = this;
  *out = mh;
  return kOk;
}
int Comm::dereg_mr(MemHandle* mh) {
  delete mh;
  return kOk;
}
int Comm::isend(const void*, size_t, int, MemHandle*, Request**) { return kErrInvalid; }
int Comm::irecv(void*, size_t, int, MemHandle*, Request**) { return kErrInvalid; }
int Comm::isend_op(const void* data, size_t size, int tag, MemHandle* mh, uint32_t op, float, Request** out) {
  if (op != 0) return kErrInvalid;          // plain transports move bytes, nothing else
  return isend(data, size, tag, mh, out);
}
int Comm::iflush(void*, size_t, MemHandle*, Request** out) {
  // Host destinations need no flush: complete immediately.
  Request* r = alloc_req(REQ_FLUSH, nullptr, 0, 0, nullptr);
  if (!r) { *out = nullptr; return kOk; }
  r->ndone.store(1, std::memory_order_release);
  *out = r;
  return kOk;
}

int Comm::free_requests() const {
  int n = 0;
  for (const Request& r : pool) n += r.in_use.load(std::memory_order_relaxed) == 0;
  return n;
}

Request* Comm::alloc_req(ReqKind k, void* buf, size_t size, int tag, MemHandle* mh) {
  uint64_t rid = next_req.fetch_add(1, std::memory_order_relaxed);
  for (int probe = 0; probe < kMaxRequests; probe++) {
    Request& r = pool[(rid + probe) % kMaxRequests];
    uint32_t z = 0;
    if (r.in_use.load(std::memory_order_relaxed) == 0 &&
        r.in_use.compare_exchange_strong(z, 1, std::memory_order_acquire)) {
      r.comm = this;
      r.kind = k;
      r.nsub.store(1, std::memory_order_relaxed);
      r.ndone.store(0, std::memory_order_relaxed);
      r.nbytes.store(0, std::memory_order_relaxed);
      r.err.store(0, std::memory_order_relaxed);
      r.buf = buf;
      r.size = size;
      r.tag = tag;
      r.mh = mh;
      r.id = rid;
      r.t_post = now_ns();
      r.prof_event = nullptr;
      r.prof_path = 0;
      memset(r.u, 0, sizeof(r.u));
      if (nvtx_on() && k != REQ_FLUSH) {
        char nm[64];
        snprintf(nm, sizeof(nm), "bnet %s-%llu %zuB", k == REQ_SEND ? "isend" : "irecv", (unsigned long long)id, size);
        r.nvtx = nvtxRangeStartA(nm);
        r.nvtx_open = true;
      }
      Telemetry& T = Telemetry::get();
      r.span = T.tracing() && k != REQ_FLUSH ? T.span_begin(k == REQ_SEND ? SPAN_ISEND : SPAN_IRECV, id, rid, size) : 0;
      if (k != REQ_FLUSH) T.m().hold_on_request.fetch_add(1, std::memory_order_relaxed);
      if (k == REQ_SEND) T.m().isend_total.fetch_add(1, std::memory_order_relaxed);
      else if (k == REQ_RECV) T.m().irecv_total.fetch_add(1, std::memory_order_relaxed);
      return &r;
    }
  }
  return nullptr;  // pool exhausted: caller returns request=NULL, NCCL retries
}

void Comm::free_req(Request* r) {
  Telemetry& T = Telemetry::get();
  if (r->prof_event) profiler_stop(r);
  if (r->nvtx_open) {
    nvtxRangeEnd(r->nvtx);
    r->nvtx_open = false;
  }
  if (r->span) T.span_end(r->span, r->nbytes.load(std::memory_order_relaxed));
  if (r->kind != REQ_FLUSH) T.m().hold_on_request.fetch_sub(1, std::memory_order_relaxed);
  r->in_use.store(0, std::memory_order_release);
}

int Comm::test(Request* r, int* done, size_t* size) {
  progress();
  int e = r->err.load(std::memory_order_acquire);
  if (e) {
    // keep the slot reserved until the comm is closed: workers may still touch it
    Telemetry::get().m().errors_total.fetch_add(1, std::memory_order_relaxed);
    *done = 0;
    return e;
  }
  if (r->complete()) {
    *done = 1;
    if (size) *size = (size_t)r->nbytes.load(std::memory_order_acquire);
    free_req(r);
  } else {
    *done = 0;
    const Config& cfg = Config::get();
    if (cfg.timeout_ms > 0 && now_ns() - r->t_post > (uint64_t)cfg.timeout_ms * 1000000ull) {
      r->fail(kErrTimeout);
      broken.store(kErrTimeout);
      return kErrTimeout;
    }
  }
  return kOk;
}

// ------------------------------------------------------------------ listen comm
ListenComm::~ListenComm() {
  if (tcp_fd >= 0) close(tcp_fd);
  if (uds_fd >= 0) close(uds_fd);
  for (auto& s : socks) close(s.fd);
  for (auto& kv : pending) {
    if (kv.second.ctrl >= 0) close(kv.second.ctrl);
    for (auto& d : kv.second.data) close(d.second);
  }
}

// ------------------------------------------------------------------ engine
Engine& Engine::get() {
  static Engine* e = new Engine();  // leaked: NCCL may call into us during static destruction
  return *e;
}

// The library starts threads (watchdog, telemetry push, TCP workers) that must never find their code unmapped: NCCL
// dlclose()s a plugin library when the last communicator goes away (and may have opened it under two names, net + tuner).
static void pin_library() {
  static bool done = false;
  if (done) return;
  done = true;
  Dl_info info;
  if (dladdr((void*)&pin_library, &info) && info.dli_fname) {
    if (!dlopen(info.dli_fname, RTLD_NOW | RTLD_NODELETE)) BNET_DEBUG("could not pin %s: %s", info.dli_fname, dlerror());
  }
}

int Engine::init() {
  std::lock_guard<std::mutex> lk(mu_);
  if (inited_) return kOk;
  pin_library();
  if (env_int("EXEC_STATS", 0) != 0) {
    // BNET_EXEC_STATS=1: one line per process at exit — how many messages the device executor moved and in how many launches
    atexit([] {
      cuda::ExecStats st;
      cuda::exec_stats(&st);
      fprintf(stderr, "[bnet stats] pid %d: %llu messages, %llu chunks, %.1f MiB, %llu kernel launches, %llu messages left in "
                      "multi-message launches\n", (int)getpid(), (unsigned long long)st.jobs, (unsigned long long)st.chunks,
              st.bytes / 1048576.0, (unsigned long long)st.launches, (unsigned long long)st.batched);
    });
  }
  const Config& cfg = Config::get();
  if (cfg.implement != "BASIC" && cfg.implement != "TOKIO") {
    // the reference returns a null backend here (src/lib.rs:20-29)
    BNET_WARN("unknown BAGUA_NET_IMPLEMENT '%s' (expected BASIC or TOKIO)", cfg.implement.c_str());
    return kErrInvalid;
  }
  // Device model (SURVEY section 5.8).  The reference has one NCCL device per NIC (reference nthread_…:241-257).
  // On an NVSwitch box the "NIC" of a GPU is its own NVLink port, so when the device path is usable every visible
  // GPU gets a virtual device of its own (guid per GPU, NVLink speed).  It carries NO pciPath: a <nic> under the GPU's
  // own <pci> node crashes NCCL's topology code, so GPUDirect is enabled by the
  // NCCL_NET_GDR_LEVEL=SYS default the plugin's init supplies instead of by PCI distance.  Every virtual device keeps a
  // TCP side on a real interface (cross-host peers, fallbacks); the plain NIC devices follow after them.
  std::vector<NetIf> nics = find_interfaces();
  cuda_ok_ = cfg.gdr && cuda::available();
  devs_.clear();
  gpu_of_dev_.clear();
  props_.clear();
  long long speed_override = env_int("SPEED_MBPS", 0);
  // grouped receives (ncclNet v5+ irecv with n > 1; csrc/plugin/plugin.cc: GroupReq): 1 = what every measured run used;
  // BNET_MAX_RECVS=8 lets NCCL aggregate the receives of grouped send/recv to one peer (not used by its all-reduce)
  int max_recvs = (int)env_int("MAX_RECVS", 1);
  if (max_recvs < 1) max_recvs = 1;
  if (max_recvs > kMaxGroupRecvs) max_recvs = kMaxGroupRecvs;
  const bool gpu_devs = env_int("GPU_DEVICES", cuda::fake() ? 0 : 1) != 0 && cfg.nvl && cuda_ok_ && !nics.empty();
  if (gpu_devs) {
    for (int g = 0; g < cuda::device_count(); g++) {
      std::string busid;
      std::string path = cuda::device_pci_path(g, &busid);
      NetIf nif = nics[(size_t)g % nics.size()];
      DeviceProps p;
      p.name = "bnet-gpu" + std::to_string(g);
      // NCCL builds its topology from pciPath: the last component must be a PCI leaf that is NOT the GPU itself (a <pci>
      // node with both a <gpu> and a <nic> child loses the GPU's link to its parent in ncclTopoAddPci).  There is no such
      // leaf for a virtual NVLink "NIC", so by default the device carries no PCI path (NCCL attaches it to the CPU, like
      // any virtual NIC) and the plugin supplies NCCL_NET_GDR_LEVEL=SYS itself (plugin.cc: tune_nccl_env), which is what
      // lets NCCL hand us device pointers.  BNET_GPU_DEVICE_PCI=gpu keeps the GPU's own path for experiments.
      static const bool own_path = env_str("GPU_DEVICE_PCI", "none") == "gpu";
      p.pci_path = own_path ? path : std::string();
      p.guid = fnv1a(busid.data(), busid.size()) ^ (uint64_t)g;
      p.ptr_support = NCCL_PTR_HOST | NCCL_PTR_CUDA;
      p.speed_mbps = speed_override > 0 ? (int)speed_override : 3600000;   // 450 GB/s per direction (H100 NVLink 4)
      p.port = 0;
      p.latency_us = 0;
      p.max_comms = 65536;
      p.max_recvs = max_recvs;
      devs_.push_back(nif);
      gpu_of_dev_.push_back(g);
      props_.push_back(p);
    }
  }
  for (size_t i = 0; i < nics.size(); i++) {
    DeviceProps p;
    p.name = nics[i].name;
    p.pci_path = nics[i].pci_path;
    p.guid = i;  // reference: guid = device index (nthread_…:250)
    p.ptr_support = NCCL_PTR_HOST | (cuda_ok_ ? NCCL_PTR_CUDA : 0);
    p.speed_mbps = nics[i].speed_mbps;
    // With the NVLink path available the "wire" is NVLink, not the NIC.
    if (cfg.nvl && cuda_ok_ && !gpu_devs) p.speed_mbps = 1600000;
    if (speed_override > 0) p.speed_mbps = (int)speed_override;
    p.port = 0;
    p.latency_us = 0;
    p.max_comms = 65536;
    p.max_recvs = max_recvs;
    devs_.push_back(nics[i]);
    gpu_of_dev_.push_back(-1);
    props_.push_back(p);
  }
  {
    std::string names;   // root span attribute like the reference's `socket_devs` (nthread_…:132-137)
    for (size_t i = 0; i < devs_.size(); i++) names += (i ? "," : "") + devs_[i].name;
    Telemetry::get().set_root_attribute(names);   // (also starts the exporters)
  }
  BNET_INFO("engine up: %zu device(s) (%d GPU-virtual + %zu NIC), implement=%s nstreams=%d min_chunksize=%zu nvl=%d cuda=%d",
            devs_.size(), gpu_devs ? cuda::device_count() : 0, nics.size(), cfg.implement.c_str(), cfg.nstreams,
            cfg.min_chunksize, cfg.nvl, (int)cuda_ok_);
  inited_ = true;
  return kOk;
}

int Engine::ndev() { return (int)devs_.size(); }

int Engine::props(int dev, DeviceProps* out) {
  if (dev < 0 || dev >= (int)props_.size()) return kErrInvalid;
  *out = props_[dev];
  return kOk;
}

int Engine::listen(int dev, void* handle_out, size_t handle_cap, ListenComm** out) {
  if (dev < 0 || dev >= (int)devs_.size() || handle_cap < sizeof(Handle)) return kErrInvalid;
  const Config& cfg = Config::get();
  const NetIf& nif = devs_[dev];
  int af = nif.addr.sa.sa_family;
  int fd = socket(af, SOCK_STREAM | SOCK_CLOEXEC, 0);
  if (fd < 0) return kErrSystem;
  SockAddr a = nif.addr;
  if (af == AF_INET) a.in4.sin_port = 0; else a.in6.sin6_port = 0;
  int one = 1;
  setsockopt(fd, SOL_SOCKET, SO_REUSEADDR, &one, sizeof(one));
  if (bind(fd, &a.sa, sockaddr_len(a)) != 0 || ::listen(fd, 16384) != 0) {  // backlog as the reference (nthread_…:101,286)
    BNET_WARN("listen: bind/listen on %s failed: %s", nif.name.c_str(), strerror(errno));
    close(fd);
    return kErrSystem;
  }
  socklen_t sl = sizeof(a);
  getsockname(fd, &a.sa, &sl);
  set_nonblocking(fd, true);

  std::unique_ptr<ListenComm> l(new ListenComm);
  l->dev = dev;
  l->tcp_fd = fd;
  Handle& h = l->handle;
  memset(&h, 0, sizeof(h));
  h.addr = a;
  if (!cfg.wire_compat) {
    h.magic = kHandleMagic;
    h.version = kWireVersion;
    h.host_hash = host_hash();
    h.listen_nonce = random_u64();
    h.pid = (uint32_t)getpid();
    h.cuda_dev = cuda_ok_ ? cuda::current_device() : -1;   // (NCCL may pick any of the equidistant virtual devices)
    if (cfg.implement == "TOKIO") h.flags |= HF_ASYNC;
    if (cfg.nvl && nvl_available()) {
      // abstract unix socket: intra-host rendezvous for the shared-memory/NVLink transport
      int ufd = socket(AF_UNIX, SOCK_STREAM | SOCK_CLOEXEC, 0);
      if (ufd >= 0) {
        sockaddr_un un{};
        un.sun_family = AF_UNIX;
        std::string name = nvl_uds_name(h.pid, h.listen_nonce);
        memcpy(un.sun_path + 1, name.data(), name.size());  // sun_path[0] = 0 -> abstract
        socklen_t ulen = (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + name.size());
        if (bind(ufd, (sockaddr*)&un, ulen) == 0 && ::listen(ufd, 1024) == 0) {
          set_nonblocking(ufd, true);
          l->uds_fd = ufd;
          h.flags |= HF_NVL;
        } else {
          close(ufd);
        }
      }
    }
  }
  memset(handle_out, 0, handle_cap);
  memcpy(handle_out, &h, sizeof(h));
  BNET_DEBUG("listen dev=%d addr=%s nvl=%d", dev, sockaddr_str(a).c_str(), (h.flags & HF_NVL) ? 1 : 0);
  *out = l.release();
  return kOk;
}

static int connect_tcp(const SockAddr& to, int timeout_ms) {
  int fd = socket(to.sa.sa_family, SOCK_STREAM | SOCK_CLOEXEC, 0);
  if (fd < 0) return -1;
  set_nonblocking(fd, true);
  int r = ::connect(fd, &to.sa, sockaddr_len(to));
  if (r != 0 && errno != EINPROGRESS) {
    close(fd);
    return -1;
  }
  if (r != 0) {
    pollfd p{fd, POLLOUT, 0};
    int pr;
    do { pr = poll(&p, 1, timeout_ms); } while (pr < 0 && errno == EINTR);
    int soerr = 0;
    socklen_t sl = sizeof(soerr);
    if (pr <= 0 || getsockopt(fd, SOL_SOCKET, SO_ERROR, &soerr, &sl) != 0 || soerr != 0) {
      close(fd);
      errno = soerr ? soerr : ETIMEDOUT;
      return -1;
    }
  }
  set_nodelay(fd);
  return fd;
}

int Engine::connect(int dev, const void* handle, Comm** out) {
  *out = nullptr;
  if (dev < 0 || dev >= (int)devs_.size()) return kErrInvalid;
  const Config& cfg = Config::get();
  Handle h;
  memcpy(&h, handle, sizeof(h));
  bool ours = h.magic == kHandleMagic && !cfg.wire_compat;
  if (ours && h.version != kWireVersion) {
    BNET_WARN("connect: peer speaks wire version %u, we speak %u", h.version, kWireVersion);
    return kErrInvalid;
  }
  // 1) same OS instance and both sides willing: shared-memory / NVLink transport
  if (ours && cfg.nvl && (h.flags & HF_NVL) && h.host_hash == host_hash() && nvl_available()) {
    Comm* c = nvl_connect(dev, h);
    if (c) {
      *out = c;
      return kOk;
    }
    BNET_INFO("connect: NVL rendezvous failed, falling back to TCP");
  }
  // 2) multi-stream TCP (reference: nthread_…:305-423 / tokio_…:336-476)
  ConnParams p;
  p.nstreams = cfg.nstreams;
  p.min_chunksize = cfg.min_chunksize;
  p.impl = cfg.implement == "TOKIO" ? 1 : 0;
  p.nonce = random_u64();
  p.compat = !ours;
  int tmo = (int)env_int("CONNECT_TIMEOUT_MS", 30000);
  std::vector<int> fds;
  int ctrl = -1;
  auto fail = [&](const char* what) {
    BNET_WARN("connect to %s failed (%s): %s", sockaddr_str(h.addr).c_str(), what, strerror(errno));
    for (int f : fds) close(f);
    if (ctrl >= 0) close(ctrl);
    return kErrSystem;
  };
  for (int i = 0; i <= p.nstreams; i++) {
    int fd = connect_tcp(h.addr, tmo);
    if (fd < 0) return fail("tcp connect");
    Preamble pre{};
    pre.stream_id_be = be64((uint64_t)i);   // i == nstreams announces the control stream
    pre.magic = kHandleMagic;
    pre.version = kWireVersion;
    pre.nstreams = (uint16_t)p.nstreams;
    pre.conn_nonce = p.nonce;
    pre.impl = (uint32_t)p.impl;
    pre.min_chunksize = (uint32_t)(p.min_chunksize > 0xffffffffull ? 0xffffffffull : p.min_chunksize);
    size_t n = p.compat ? sizeof(uint64_t) : sizeof(pre);
    if (write_all(fd, &pre, n, nullptr, tmo) != kOk) {
      close(fd);
      return fail("preamble");
    }
    if (i < p.nstreams) fds.push_back(fd); else ctrl = fd;
  }
  Comm* c = p.impl ? tcp_async_make_send(dev, ctrl, fds, p) : tcp_threads_make_send(dev, ctrl, fds, p);
  if (!c) return kErrInternal;
  *out = c;
  return kOk;
}

int Engine::accept(ListenComm* l, Comm** out, bool blocking) {
  *out = nullptr;
  const Config& cfg = Config::get();
  bool compat = l->handle.magic != kHandleMagic;
  uint64_t t0 = now_ns();
  for (;;) {
    std::unique_lock<std::mutex> lk(l->mu);
    // (1) take every connection the kernel has queued
    for (int which = 0; which < 2; which++) {
      int lfd = which ? l->uds_fd : l->tcp_fd;
      if (lfd < 0) continue;
      for (;;) {
        int fd = accept4(lfd, nullptr, nullptr, SOCK_NONBLOCK | SOCK_CLOEXEC);
        if (fd < 0) {
          if (errno == EINTR) continue;
          if (errno != EAGAIN && errno != EWOULDBLOCK) BNET_WARN("accept4: %s", strerror(errno));
          break;
        }
        if (!which) set_nodelay(fd);
        ListenComm::Sock s{};
        s.fd = fd;
        s.uds = which == 1;
        s.got = 0;
        l->socks.push_back(s);
      }
    }
    // (2) read preambles without blocking
    for (size_t i = 0; i < l->socks.size();) {
      ListenComm::Sock& s = l->socks[i];
      size_t need = s.uds ? nvl_hello_size() : (compat ? sizeof(uint64_t) : sizeof(Preamble));
      bool drop = false, ready = false;
      while (s.got < need) {
        ssize_t r = recv(s.fd, s.buf + s.got, need - s.got, 0);
        if (r > 0) { s.got += (size_t)r; continue; }
        if (r == 0) { drop = true; break; }
        if (errno == EINTR) continue;
        if (errno != EAGAIN && errno != EWOULDBLOCK) drop = true;
        break;
      }
      if (s.got == need) ready = true;
      if (drop) {
        close(s.fd);
        l->socks.erase(l->socks.begin() + i);
        continue;
      }
      if (!ready) { i++; continue; }
      ListenComm::Sock done = s;
      l->socks.erase(l->socks.begin() + i);
      if (done.uds) {
        Comm* c = nvl_accept(l->dev, done.fd, done.buf, need);
        if (!c) { close(done.fd); continue; }
        *out = c;
        return kOk;
      }
      Preamble pre{};
      memcpy(&pre, done.buf, need);
      uint64_t sid = be64(pre.stream_id_be);
      uint64_t nonce = 0;
      ConnParams p;
      if (compat) {
        p.nstreams = cfg.nstreams;
        p.min_chunksize = cfg.min_chunksize;
        p.impl = cfg.implement == "TOKIO" ? 1 : 0;
        p.nonce = 0;
        p.compat = true;
      } else {
        if (pre.magic != kHandleMagic || pre.version != kWireVersion || pre.nstreams == 0) {
          BNET_WARN("accept: bad preamble (magic %x version %u), dropping socket", pre.magic, pre.version);
          close(done.fd);
          continue;
        }
        nonce = pre.conn_nonce;
        p.nstreams = pre.nstreams;
        p.min_chunksize = pre.min_chunksize;
        p.impl = (int)pre.impl;
        p.nonce = nonce;
        p.compat = false;
      }
      ListenComm::Pending& pd = l->pending[nonce];
      pd.p = p;
      if (sid == (uint64_t)p.nstreams) {
        if (pd.ctrl >= 0) close(pd.ctrl);
        pd.ctrl = done.fd;
      } else if (sid < (uint64_t)p.nstreams) {
        pd.data[(int)sid] = done.fd;
      } else {
        BNET_WARN("accept: stream id %llu out of range (nstreams %d)", (unsigned long long)sid, p.nstreams);
        close(done.fd);
      }
    }
    // (3) a complete group becomes a recv comm (reference: nthread_…:425-522)
    for (auto it = l->pending.begin(); it != l->pending.end(); ++it) {
      ListenComm::Pending& pd = it->second;
      if (pd.ctrl >= 0 && (int)pd.data.size() == pd.p.nstreams) {
        std::vector<int> fds;
        for (auto& kv : pd.data) fds.push_back(kv.second);  // ordered by stream id
        int ctrl = pd.ctrl;
        ConnParams p = pd.p;
        l->pending.erase(it);
        Comm* c = p.impl ? tcp_async_make_recv(l->dev, ctrl, fds, p) : tcp_threads_make_recv(l->dev, ctrl, fds, p);
        if (!c) return kErrInternal;
        *out = c;
        return kOk;
      }
    }
    lk.unlock();
    if (!blocking) return kOk;
    int tmo = (int)env_int("ACCEPT_TIMEOUT_MS", 0);
    if (tmo > 0 && now_ns() - t0 > (uint64_t)tmo * 1000000ull) return kErrTimeout;
    pollfd pf[64];
    int n = 0;
    pf[n++] = pollfd{l->tcp_fd, POLLIN, 0};
    if (l->uds_fd >= 0) pf[n++] = pollfd{l->uds_fd, POLLIN, 0};
    {
      std::lock_guard<std::mutex> lk2(l->mu);
      for (auto& s : l->socks)
        if (n < 64) pf[n++] = pollfd{s.fd, POLLIN, 0};
    }
    poll(pf, n, 20);
  }
}

}  // namespace bnet

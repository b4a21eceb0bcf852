// NCCL ext-net ABI shims: one exported table per ABI version, all delegating to
// the engine.  Counterpart of the reference's L1 (reference:
// cc/v4/nccl_net_v4.cc:1-226, cc/v3/nccl_net_v3.cc:1-226) — but the installed
// NCCL 2.27/2.28 only probe v6..v11, so v6+ tables are what NCCL actually loads;
// v3/v4 keep the reference's symbols alive (and drive our own loopback harness).
//
// Semantics that differ from the reference on purpose:
//   * regMr accepts NCCL_PTR_CUDA when the CUDA side is usable and always writes
//     *mhandle (the reference rejects CUDA and leaves *mhandle unset, :105-109)
//   * iflush works (device-side fence / no-op for host memory) instead of
//     returning ncclInternalError (:145-149)
//   * v5+ connect/accept never block on the peer: they return *comm == NULL
//     until the connection is ready
#include <stdlib.h>

#include <deque>
#include <string.h>

#include "bnet/nccl_net_abi.h"
#include "core/engine.h"
#include "core/telemetry.h"
#include "plugin/plugin_shims.h"

using namespace bnet;

#define BNET_EXPORT __attribute__((visibility("default")))
#pragma GCC diagnostic ignored "-Wunused-function"

namespace {

const char kName[] = "BNet";

// strings handed to NCCL must stay alive: cache per device
struct PropStrings {
  std::string name, pci;
};
// (a deque: growing it never moves the strings NCCL already holds pointers into — short names live INSIDE the
//  std::string object, so a reallocating vector would leave NCCL with dangling name pointers)
std::deque<PropStrings>& prop_cache() {
  static std::deque<PropStrings>* v = new std::deque<PropStrings>();
  return *v;
}
std::mutex g_prop_mu;

ncclResult_t fill_common(int dev, DeviceProps* p, char** name, char** pci) {
  int st = Engine::get().props(dev, p);
  if (st) return to_nccl(st);
  std::lock_guard<std::mutex> lk(g_prop_mu);
  auto& c = prop_cache();
  if ((int)c.size() <= dev) c.resize(dev + 1);
  if (c[dev].name != p->name) c[dev].name = p->name;          // (unchanged strings keep their buffers)
  if (c[dev].pci != p->pci_path) c[dev].pci = p->pci_path;
  *name = const_cast<char*>(c[dev].name.c_str());
  *pci = c[dev].pci.empty() ? nullptr : const_cast<char*>(c[dev].pci.c_str());
  return ncclSuccess;
}

// NCCL drives a net plugin through a proxy pipeline of NCCL_BUFFSIZE/8-byte slices per channel, and for small and
// medium messages it prefers the LL protocol, whose buffers live in host memory (so they ride our shared-memory
// ring, not NVLink).  Over this transport the measured optimum is the Simple protocol with large slices and many
// channels.  NCCL reads these variables after the plugin's init(), so a default can
// be supplied here; anything the user has set wins, BNET_TUNE_NCCL=0 leaves the environment alone.
void tune_nccl_env() {
  if (env_int("TUNE_NCCL", 1) == 0) return;
  const Config& cfg = Config::get();
  if (!cfg.nvl || !cfg.gdr || !Engine::get().cuda_ok()) return;
  struct KV { const char* k; const char* v; };
  static const KV defaults[] = {
      {"NCCL_PROTO", "Simple"},
      {"NCCL_BUFFSIZE", "33554432"},
      {"NCCL_MIN_NCHANNELS", "16"},
      // our "NIC" is the GPU's own NVLink port: device pointers are welcome wherever NCCL's topology puts the device
      {"NCCL_NET_GDR_LEVEL", "SYS"},
      {"NCCL_NET_GDR_READ", "1"},
  };
  {
    const char* ml = getenv("CUDA_MODULE_LOADING");
    if (!ml || strcmp(ml, "EAGER"))
      BNET_INFO("CUDA_MODULE_LOADING is not EAGER: a kernel the application launches for the FIRST time while a collective is in "
                "flight makes CUDA's lazy loader wait for the device, and the collective waits for this transport's kernels "
                "behind it (dead-lock).  Either launch every kernel of a step once before the first collective (a warm-up "
                "step without the process group), or export CUDA_MODULE_LOADING=EAGER before the process starts and pay "
                "its start-up time (`python -m bagua_net_b200.utils.env` prints the full environment).");
  }
  // with our tuner plugin in charge (NCCL_TUNER_PLUGIN=bnet) LL stays available — the tuner confines it to tiny messages
  // — but LL128 is excluded either way (it needs a 128-byte store atomicity a copy kernel does not preserve)
  const char* tp = getenv("NCCL_TUNER_PLUGIN");
  const bool our_tuner = tp && strstr(tp, "bnet") && env_int("TUNER", 1) != 0;
  for (const KV& d : defaults)
    if (!getenv(d.k)) {
      const char* v = (!strcmp(d.k, "NCCL_PROTO") && our_tuner) ? "LL,Simple" : d.v;
      setenv(d.k, v, 0);
      if (!strcmp(d.k, "NCCL_PROTO")) setenv("BNET_PROTO_DEFAULTED", "1", 1);
      BNET_INFO("init: %s=%s (transport default; set it yourself or BNET_TUNE_NCCL=0 to override)", d.k, v);
    }
}

ncclResult_t do_init(ncclDebugLogger_t logfn) {
  if (logfn) log_set_nccl_logger(logfn);
  int st = Engine::get().init();
  if (st) BNET_WARN("init failed: %s", status_str(st));
  else tune_nccl_env();
  return to_nccl(st);
}

ncclResult_t do_devices(int* ndev) {
  if (!ndev) return ncclInvalidArgument;
  *ndev = Engine::get().ndev();
  return ncclSuccess;
}

ncclResult_t do_listen(int dev, void* handle, size_t cap, void** lcomm) {
  CallScope cs_("listen");
  ListenComm* l = nullptr;
  int st = Engine::get().listen(dev, handle, cap, &l);
  if (st) {
    BNET_WARN("listen(dev=%d) failed: %s", dev, status_str(st));
    return to_nccl(st);
  }
  *lcomm = l;
  return ncclSuccess;
}

ncclResult_t do_connect(int dev, void* handle, void** scomm) {
  CallScope cs_("connect");
  Comm* c = nullptr;
  int st = Engine::get().connect(dev, handle, &c);
  if (st) {
    BNET_WARN("connect(dev=%d) failed: %s", dev, status_str(st));
    return to_nccl(st);
  }
  *scomm = c;
  BNET_TRACE("connect dev=%d -> comm %p (%s)", dev, (void*)c, c ? c->transport() : "pending");
  return ncclSuccess;
}

ncclResult_t do_accept(void* lcomm, void** rcomm, bool blocking) {
  CallScope cs_("accept");
  if (!lcomm) return ncclInvalidArgument;
  Comm* c = nullptr;
  int st = Engine::get().accept(static_cast<ListenComm*>(lcomm), &c, blocking);
  if (st) {
    BNET_WARN("accept failed: %s", status_str(st));
    return to_nccl(st);
  }
  *rcomm = c;
  if (c) BNET_TRACE("accept -> comm %p (%s)", (void*)c, c->transport());
  return ncclSuccess;
}

ncclResult_t do_regmr(void* comm, void* data, size_t size, int type, void** mhandle) {
  CallScope cs_("regMr");
  if (!comm || !mhandle) return ncclInvalidArgument;
  MemHandle* mh = nullptr;
  int st = static_cast<Comm*>(comm)->reg_mr(data, size, type, &mh);
  if (st) {
    BNET_WARN("regMr(%p, %zu, type=%d) failed: %s", data, size, type, status_str(st));
    return to_nccl(st);
  }
  *mhandle = mh;
  return ncclSuccess;
}

ncclResult_t do_deregmr(void* comm, void* mhandle) {
  CallScope cs_("deregMr");
  if (!comm) return ncclInvalidArgument;
  if (!mhandle) return ncclSuccess;
  return to_nccl(static_cast<Comm*>(comm)->dereg_mr(static_cast<MemHandle*>(mhandle)));
}

ncclResult_t do_isend(void* scomm, void* data, size_t size, int tag, void* mh, void** request) {
  CallScope cs_("isend");
  if (!scomm || !request) return ncclInvalidArgument;
  Request* r = nullptr;
  int st = static_cast<Comm*>(scomm)->isend(data, size, tag, static_cast<MemHandle*>(mh), &r);
  if (st) {
    BNET_WARN("isend(%zu bytes) failed: %s", size, status_str(st));
    return to_nccl(st);
  }
  *request = r;
  BNET_TRACE("isend comm=%p data=%p size=%zu req=%p", scomm, data, size, (void*)r);
  return ncclSuccess;
}

ncclResult_t do_irecv(void* rcomm, void* data, size_t size, int tag, void* mh, void** request) {
  CallScope cs_("irecv");
  if (!rcomm || !request) return ncclInvalidArgument;
  Request* r = nullptr;
  int st = static_cast<Comm*>(rcomm)->irecv(data, size, tag, static_cast<MemHandle*>(mh), &r);
  if (st) {
    BNET_WARN("irecv(%zu bytes) failed: %s", size, status_str(st));
    return to_nccl(st);
  }
  *request = r;
  BNET_TRACE("irecv comm=%p data=%p size=%zu req=%p", rcomm, data, size, (void*)r);
  return ncclSuccess;
}

ncclResult_t do_iflush(void* rcomm, void* data, size_t size, void* mh, void** request) {
  CallScope cs_("iflush");
  if (!rcomm || !request) return ncclInvalidArgument;
  Request* r = nullptr;
  int st = static_cast<Comm*>(rcomm)->iflush(data, size, static_cast<MemHandle*>(mh), &r);
  if (st) return to_nccl(st);
  *request = r;
  return ncclSuccess;
}

// A grouped receive (ncclNet v5+: irecv with n > 1 — NCCL aggregates the receives of grouped send/recv to one peer and
// gives every entry of a group the SAME tag, the sender's rank) is n ordinary receives matched, in posting order, to the
// next n isends of the connection: exactly what the transports' FIFO matching delivers.  The parent lives on the heap for
// the lifetime of the group; `magic` sits where a Request keeps its in_use word (0 / 1), which is how test() tells them apart.
struct GroupReq {
  uint32_t magic;
  int n;
  Request* sub[kMaxGroupRecvs];
  int sizes[kMaxGroupRecvs];
  bool fin[kMaxGroupRecvs];
  int err;
};
constexpr uint32_t kGroupMagic = 0x47525051u;   // "GRPQ"
static_assert(offsetof(Request, in_use) == 0, "GroupReq::magic must overlay Request::in_use");

ncclResult_t do_irecv_group(void* rcomm, int n, void** data, const size_t* sizes, int* tags, void** mhs, void** request) {
  CallScope cs_("irecv(group)");
  if (!rcomm || !request || !data || !sizes || n < 1) return ncclInvalidArgument;
  if (n > kMaxGroupRecvs) return ncclInvalidUsage;
  *request = nullptr;
  Comm* c = static_cast<Comm*>(rcomm);
  if (c->free_requests() < n) return ncclSuccess;            // all of the group or nothing: NCCL retries
  GroupReq* g = new GroupReq();
  g->magic = kGroupMagic;
  g->n = n;
  for (int i = 0; i < n; i++) {
    Request* r = nullptr;
    int st = c->irecv(data[i], sizes[i], tags ? tags[i] : 0, mhs ? static_cast<MemHandle*>(mhs[i]) : nullptr, &r);
    if (st || !r) {
      // part of the group is posted and cannot be taken back: the connection is unusable from here on
      BNET_WARN("irecv group: entry %d of %d could not be posted (%s)", i, n, st ? status_str(st) : "request pool exhausted");
      c->broken.store(st ? st : kErrInternal, std::memory_order_release);
      delete g;
      return st ? to_nccl(st) : ncclInternalError;
    }
    g->sub[i] = r;
  }
  *request = g;
  return ncclSuccess;
}

ncclResult_t test_group(GroupReq* g, int* done, int* sizes) {
  *done = 0;
  bool all = true;
  for (int i = 0; i < g->n; i++) {
    if (g->fin[i]) continue;
    int d = 0;
    size_t sz = 0;
    int st = g->sub[i]->comm->test(g->sub[i], &d, &sz);
    if (st) {
      BNET_WARN("test: entry %d of a grouped receive failed: %s", i, status_str(st));
      g->fin[i] = true;                  // (a failed request has been released by the transport)
      g->err = st;
      continue;
    }
    if (d) { g->fin[i] = true; g->sizes[i] = (int)sz; } else all = false;
  }
  if (!all) return ncclSuccess;
  const int err = g->err;
  if (!err) {
    *done = 1;
    if (sizes) for (int i = 0; i < g->n; i++) sizes[i] = g->sizes[i];
  }
  delete g;
  return err ? to_nccl(err) : ncclSuccess;
}

ncclResult_t do_test(void* request, int* done, int* size) {
  CallScope cs_("test");
  if (!request || !done) return ncclInvalidArgument;
  if (*static_cast<uint32_t*>(request) == kGroupMagic) return test_group(static_cast<GroupReq*>(request), done, size);
  Request* r = static_cast<Request*>(request);
  size_t sz = 0;
  int st = r->comm->test(r, done, &sz);
  if (st) {
    BNET_WARN("test: request %llu on %s comm failed: %s", (unsigned long long)r->id, r->comm->transport(),
              status_str(st));
    return to_nccl(st);
  }
  if (*done && size) *size = (int)sz;
  return ncclSuccess;
}

ncclResult_t do_close(void* comm) {
  CallScope cs_("close");
  delete static_cast<Comm*>(comm);
  return ncclSuccess;
}

// ---- v3 / v4 (blocking accept like the reference; int sizes; 64-byte handle) --------
ncclResult_t v4_init(ncclDebugLogger_t f) { return do_init(f); }
ncclResult_t v4_props(int dev, ncclNetProperties_v4_t* o) {
  DeviceProps p;
  ncclResult_t r = fill_common(dev, &p, &o->name, &o->pciPath);
  if (r) return r;
  o->guid = p.guid;
  o->ptrSupport = p.ptr_support;
  o->speed = p.speed_mbps;
  o->port = p.port;
  o->maxComms = p.max_comms;
  return ncclSuccess;
}
ncclResult_t v4_listen(int dev, void* h, void** l) { return do_listen(dev, h, NCCL_NET_HANDLE_MAXSIZE_V4, l); }
ncclResult_t v4_connect(int dev, void* h, void** s) { return do_connect(dev, h, s); }
ncclResult_t v4_accept(void* l, void** r) { return do_accept(l, r, /*blocking=*/true); }
ncclResult_t v4_regmr(void* c, void* d, int size, int type, void** mh) { return do_regmr(c, d, (size_t)size, type, mh); }
// v3/v4: "may return request == NULL if the call cannot be performed (or would block)" — NCCL retries.  The reference never
// does (its queues are unbounded); here a full request pool says so instead of holding NCCL's proxy thread in a spin.
ncclResult_t v4_isend(void* c, void* d, int size, void* mh, void** req) { return do_isend(c, d, (size_t)size, 0, mh, req); }
ncclResult_t v4_irecv(void* c, void* d, int size, void* mh, void** req) { return do_irecv(c, d, (size_t)size, 0, mh, req); }
ncclResult_t v4_iflush(void* c, void* d, int size, void* mh, void** req) { return do_iflush(c, d, (size_t)size, mh, req); }
ncclResult_t v3_flush(void* c, void* d, int size, void* mh) {
  void* req = nullptr;
  ncclResult_t r = do_iflush(c, d, (size_t)size, mh, &req);
  if (r) return r;
  int done = 0;
  while (req && !done) {
    r = do_test(req, &done, nullptr);
    if (r) return r;
  }
  return ncclSuccess;
}

// ---- v5..v8 -----------------------------------------------------------------------
template <typename P>
ncclResult_t props_v6like(int dev, P* o) {
  DeviceProps p;
  ncclResult_t r = fill_common(dev, &p, &o->name, &o->pciPath);
  if (r) return r;
  o->guid = p.guid;
  o->ptrSupport = p.ptr_support;
  o->speed = p.speed_mbps;
  o->port = p.port;
  o->latency = p.latency_us;
  o->maxComms = p.max_comms;
  o->maxRecvs = p.max_recvs;
  return ncclSuccess;
}
}  // namespace

// (shared with the CollNet tables of csrc/plugin/collnet.cc: csrc/plugin/plugin_shims.h)
namespace bnet {
namespace plugin {
ncclResult_t init(ncclDebugLogger_t logfn) { return do_init(logfn); }
ncclResult_t v4_props(int dev, ncclNetProperties_v4_t* o) { return ::v4_props(dev, o); }
ncclResult_t v6_props(int dev, ncclNetProperties_v6_t* o) { return props_v6like(dev, o); }
ncclResult_t v7_props(int dev, ncclNetProperties_v7_t* o) {
  ncclResult_t r = props_v6like(dev, o);
  o->netDeviceType = NCCL_NET_DEVICE_HOST;
  o->netDeviceVersion = NCCL_NET_DEVICE_INVALID_VERSION;
  return r;
}
ncclResult_t v8_props(int dev, ncclNetProperties_v8_t* o) {
  ncclResult_t r = props_v6like(dev, o);
  o->regIsGlobal = 0;
  o->netDeviceType = NCCL_NET_DEVICE_HOST;
  o->netDeviceVersion = NCCL_NET_DEVICE_INVALID_VERSION;
  return r;
}
ncclResult_t v9_props(int dev, ncclNetProperties_v9_t* o) {
  ncclResult_t r = props_v6like(dev, o);
  o->regIsGlobal = 0;
  o->forceFlush = 0;
  o->netDeviceType = NCCL_NET_DEVICE_HOST;
  o->netDeviceVersion = NCCL_NET_DEVICE_INVALID_VERSION;
  o->vProps.ndevs = 1;
  o->vProps.devs[0] = dev;
  o->maxP2pBytes = (size_t)1 << 40;
  o->maxCollBytes = (size_t)1 << 40;
  return r;
}
}  // namespace plugin
}  // namespace bnet

namespace {
using bnet::plugin::v6_props;
using bnet::plugin::v7_props;
using bnet::plugin::v8_props;
using bnet::plugin::v9_props;

ncclResult_t v6_listen(int dev, void* h, void** l) { return do_listen(dev, h, NCCL_NET_HANDLE_MAXSIZE, l); }
ncclResult_t v6_connect(int dev, void* h, void** s) { return do_connect(dev, h, s); }
ncclResult_t v6_accept(void* l, void** r) { return do_accept(l, r, /*blocking=*/false); }
ncclResult_t v7_connect(int dev, void* h, void** s, ncclNetDeviceHandle_v7_t** dh) {
  if (dh) *dh = nullptr;
  return do_connect(dev, h, s);
}
ncclResult_t v7_accept(void* l, void** r, ncclNetDeviceHandle_v7_t** dh) {
  if (dh) *dh = nullptr;
  return do_accept(l, r, false);
}
ncclResult_t v10_connect(int dev, ncclNetCommConfig_v10_t*, void* h, void** s, ncclNetDeviceHandle_v10_t** dh) {
  if (dh) *dh = nullptr;
  return do_connect(dev, h, s);
}
ncclResult_t v6_regmr(void* c, void* d, int size, int type, void** mh) { return do_regmr(c, d, (size_t)size, type, mh); }
ncclResult_t v8_regmr(void* c, void* d, size_t size, int type, void** mh) { return do_regmr(c, d, size, type, mh); }
ncclResult_t v6_regmr_dmabuf(void* c, void* d, size_t size, int type, uint64_t, int, void** mh) {
  return do_regmr(c, d, size, type, mh);   // we never advertise NCCL_PTR_DMABUF; treat as plain regMr
}
ncclResult_t v6_isend(void* c, void* d, int size, int tag, void* mh, void** req) { return do_isend(c, d, (size_t)size, tag, mh, req); }
ncclResult_t v9_isend(void* c, void* d, size_t size, int tag, void* mh, void** req) { return do_isend(c, d, size, tag, mh, req); }
ncclResult_t v10_isend(void* c, void* d, size_t size, int tag, void* mh, void* ph, void** req) {
  ncclResult_t r = do_isend(c, d, size, tag, mh, req);
  if (r == ncclSuccess && *req && ph) profiler_start(static_cast<Request*>(*req), ph);
  return r;
}
ncclResult_t v6_irecv(void* c, int n, void** data, int* sizes, int* tags, void** mhs, void** req) {
  if (n == 1) return do_irecv(c, data[0], (size_t)sizes[0], tags ? tags[0] : 0, mhs ? mhs[0] : nullptr, req);
  if (n < 1 || n > kMaxGroupRecvs || !sizes) return ncclInvalidUsage;
  size_t sz[kMaxGroupRecvs];
  for (int i = 0; i < n; i++) sz[i] = (size_t)sizes[i];
  return do_irecv_group(c, n, data, sz, tags, mhs, req);
}
ncclResult_t v9_irecv(void* c, int n, void** data, size_t* sizes, int* tags, void** mhs, void** req) {
  if (n == 1) return do_irecv(c, data[0], sizes[0], tags ? tags[0] : 0, mhs ? mhs[0] : nullptr, req);
  return do_irecv_group(c, n, data, sizes, tags, mhs, req);
}
ncclResult_t v10_irecv(void* c, int n, void** data, size_t* sizes, int* tags, void** mhs, void** phs, void** req) {
  ncclResult_t r = v9_irecv(c, n, data, sizes, tags, mhs, req);
  if (r == ncclSuccess && *req && phs) {
    if (n == 1) {
      if (phs[0]) profiler_start(static_cast<Request*>(*req), phs[0]);
    } else {
      GroupReq* g = static_cast<GroupReq*>(*req);
      for (int i = 0; i < n; i++)
        if (phs[i]) profiler_start(g->sub[i], phs[i]);
    }
  }
  return r;
}
// one flush covers a group: the sender's kernel has fenced every entry before its completion word became visible
ncclResult_t v6_iflush(void* c, int n, void** data, int* sizes, void** mhs, void** req) {
  if (n < 1 || n > kMaxGroupRecvs) return ncclInvalidUsage;
  return do_iflush(c, data[0], (size_t)sizes[0], mhs ? mhs[0] : nullptr, req);
}
ncclResult_t v7_get_device_mr(void*, void*, void**) { return ncclInternalError; }
ncclResult_t v7_irecv_consumed(void*, int, void*) { return ncclSuccess; }
ncclResult_t v10_init(ncclDebugLogger_t f, ncclProfilerCallback_t prof) {
  profiler_set_callback(prof);   // events of ours inside NCCL's profiler: include/bnet/bnet_profiler.h
  return do_init(f);
}

}  // namespace

// ---- exported tables -----------------------------------------------------------------
extern "C" {
BNET_EXPORT ncclNet_v3_t ncclNetPlugin_v3 = {
    kName, v4_init, do_devices, v4_props, v4_listen, v4_connect, v4_accept, v4_regmr, do_deregmr,
    v4_isend, v4_irecv, v3_flush, do_test, do_close, do_close, do_close};

BNET_EXPORT ncclNet_v4_t ncclNetPlugin_v4 = {
    kName, v4_init, do_devices, v4_props, v4_listen, v4_connect, v4_accept, v4_regmr, do_deregmr,
    v4_isend, v4_irecv, v4_iflush, do_test, do_close, do_close, do_close};

BNET_EXPORT ncclNet_v5_t ncclNetPlugin_v5 = {
    kName, v4_init, do_devices, v6_props, v6_listen, v6_connect, v6_accept, v6_regmr, do_deregmr,
    v6_isend, v6_irecv, v6_iflush, do_test, do_close, do_close, do_close};

BNET_EXPORT ncclNet_v6_t ncclNetPlugin_v6 = {
    kName, v4_init, do_devices, v6_props, v6_listen, v6_connect, v6_accept, v6_regmr, v6_regmr_dmabuf,
    do_deregmr, v6_isend, v6_irecv, v6_iflush, do_test, do_close, do_close, do_close};

BNET_EXPORT ncclNet_v7_t ncclNetPlugin_v7 = {
    kName, v4_init, do_devices, v7_props, v6_listen, v7_connect, v7_accept, v6_regmr, v6_regmr_dmabuf,
    do_deregmr, v6_isend, v6_irecv, v6_iflush, do_test, do_close, do_close, do_close,
    v7_get_device_mr, v7_irecv_consumed};

BNET_EXPORT ncclNet_v8_t ncclNetPlugin_v8 = {
    kName, v4_init, do_devices, v8_props, v6_listen, v7_connect, v7_accept, v8_regmr, v6_regmr_dmabuf,
    do_deregmr, v6_isend, v6_irecv, v6_iflush, do_test, do_close, do_close, do_close,
    v7_get_device_mr, v7_irecv_consumed};

#ifdef BNET_EXPORT_V9_V10
BNET_EXPORT ncclNet_v9_t ncclNetPlugin_v9 = {
    kName, v4_init, do_devices, v9_props, v6_listen, v7_connect, v7_accept, v8_regmr, v6_regmr_dmabuf,
    do_deregmr, v9_isend, v9_irecv, v6_iflush, do_test, do_close, do_close, do_close,
    v7_get_device_mr, v7_irecv_consumed, nullptr};

BNET_EXPORT ncclNet_v10_t ncclNetPlugin_v10 = {
    kName, v10_init, do_devices, v9_props, v6_listen, v10_connect, v7_accept, v8_regmr, v6_regmr_dmabuf,
    do_deregmr, v10_isend, v10_irecv, v6_iflush, do_test, do_close, do_close, do_close,
    v7_get_device_mr, v7_irecv_consumed, nullptr};
#endif
}  // extern "C"

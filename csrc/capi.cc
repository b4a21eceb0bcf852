// Plain-C entry points for the Python package and the tests (ctypes).  The NCCL
// plugin tables live in plugin/plugin.cc; this file exposes the utilities the
// reference unit-tests (reference: src/utils.rs:263-314) plus telemetry access.
#include <string.h>

#include <sstream>

#include "core/engine.h"
#include "core/netif.h"
#include "core/telemetry.h"
#include "cuda/cuda_iface.h"
#include "cuda/nvl_exec.h"

using namespace bnet;

#define BNET_API extern "C" __attribute__((visibility("default")))

static int copy_out(const std::string& s, char* out, int cap) {
  if (!out || cap <= 0) return (int)s.size();
  int n = (int)s.size() < cap - 1 ? (int)s.size() : cap - 1;
  memcpy(out, s.data(), n);
  out[n] = 0;
  return (int)s.size();
}

BNET_API const char* bnet_version() { return "bnet 0.2 (sm_90a)"; }

BNET_API unsigned long long bnet_chunk_size(unsigned long long total, unsigned long long min_chunk,
                                            unsigned long long nchunks) {
  return chunk_size(total, min_chunk, nchunks);
}
BNET_API unsigned long long bnet_chunk_count(unsigned long long total, unsigned long long min_chunk,
                                             unsigned long long nchunks) {
  return chunk_count(total, chunk_size(total, min_chunk, nchunks));
}

BNET_API int bnet_parse_user_pass_addr(const char* raw, char* user, char* pass, char* addr, int cap) {
  UserPassAddr u;
  if (!parse_user_pass_and_addr(raw ? raw : "", &u)) return -1;
  copy_out(u.user, user, cap);
  copy_out(u.pass, pass, cap);
  copy_out(u.addr, addr, cap);
  return 0;
}

BNET_API int bnet_sockaddr_roundtrip(const char* in, char* out, int cap) {
  SockAddr a;
  if (!sockaddr_parse(in, &a)) return -1;
  // through the 64-byte NCCL handle and back, like the reference's test_socket_handle
  Handle h{};
  h.addr = a;
  unsigned char wire[NCCL_NET_HANDLE_MAXSIZE_V4];
  memset(wire, 0, sizeof(wire));
  memcpy(wire, &h, sizeof(h));
  Handle back;
  memcpy(&back, wire, sizeof(back));
  copy_out(sockaddr_str(back.addr), out, cap);
  return 0;
}

BNET_API int bnet_base64(const char* in, char* out, int cap) { return copy_out(base64(in ? in : ""), out, cap); }

BNET_API int bnet_if_filter_accepts(const char* spec, const char* ifname) {
  return IfFilter::parse(spec ? spec : "").accepts(ifname ? ifname : "") ? 1 : 0;
}

// JSON list of {"name","addr","pci","speed","loopback"}
BNET_API int bnet_find_interfaces(const char* spec, int family, char* out, int cap) {
  std::vector<NetIf> v = find_interfaces(spec && *spec ? spec : nullptr, family);
  std::ostringstream o;
  o << "[";
  for (size_t i = 0; i < v.size(); i++) {
    if (i) o << ",";
    o << "{\"name\":\"" << v[i].name << "\",\"addr\":\"" << sockaddr_str(v[i].addr) << "\",\"pci\":\"" << v[i].pci_path
      << "\",\"speed\":" << v[i].speed_mbps << ",\"loopback\":" << (v[i].loopback ? "true" : "false") << "}";
  }
  o << "]";
  return copy_out(o.str(), out, cap);
}

BNET_API void bnet_config_reload() { Config::reload(); }

BNET_API int bnet_config_json(char* out, int cap) {
  const Config& c = Config::get();
  std::ostringstream o;
  o << "{\"implement\":\"" << c.implement << "\",\"nstreams\":" << c.nstreams << ",\"min_chunksize\":" << c.min_chunksize
    << ",\"async_workers\":" << c.async_workers << ",\"rank\":" << c.rank << ",\"nvl\":" << c.nvl << ",\"gdr\":" << c.gdr
    << ",\"wire_compat\":" << c.wire_compat << ",\"timeout_ms\":" << c.timeout_ms
    << ",\"shm_ring_bytes\":" << c.shm_ring_bytes << "}";
  return copy_out(o.str(), out, cap);
}

BNET_API int bnet_metrics_text(char* out, int cap) { return copy_out(Telemetry::get().render_prometheus(), out, cap); }
BNET_API int bnet_trace_json(char* out, int cap) { return copy_out(Telemetry::get().render_trace_json(), out, cap); }
BNET_API int bnet_telemetry_flush() { return Telemetry::get().flush(); }
// the collector wire formats, rendered from the beginning of the span ring (tests decode them)
BNET_API int bnet_trace_jaeger_thrift(char* out, int cap) {
  uint64_t cur = 0;
  std::string b = Telemetry::get().render_jaeger_thrift(&cur);
  if ((int)b.size() > cap) return -1;
  memcpy(out, b.data(), b.size());
  return (int)b.size();
}
BNET_API int bnet_trace_otlp_json(char* out, int cap) {
  uint64_t cur = 0;
  return copy_out(Telemetry::get().render_otlp_json(&cur), out, cap);
}
BNET_API int bnet_http_send(const char* method, const char* hostport, const char* path, const char* body,
                            const char* user, const char* pass) {
  return Telemetry::http_send(method, hostport, path, "text/plain", body ? body : "", user ? user : "", pass ? pass : "", 1000);
}

BNET_API int bnet_cuda_available() { return cuda::available() ? 1 : 0; }
BNET_API int bnet_cuda_fake() { return cuda::fake() ? 1 : 0; }

BNET_API int bnet_exec_stats(unsigned long long* out5) {
  cuda::ExecStats s;
  cuda::exec_stats(&s);
  out5[0] = s.jobs; out5[1] = s.chunks; out5[2] = s.bytes; out5[3] = s.launches; out5[4] = s.persistent;
  return 0;
}

BNET_API const char* bnet_comm_transport(void* comm) { return comm ? static_cast<Comm*>(comm)->transport() : ""; }

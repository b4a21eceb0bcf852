// Narrow interface between the host engine (plain C++) and the CUDA side
// (runtime + driver API + sm_90a kernels).  Everything degrades to "not
// available" on a box without a GPU/driver so the TCP + shared-memory paths and
// all CPU tests keep working.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>

namespace bnet {
namespace cuda {

bool available();                 // a usable CUDA device exists in this process
bool fake();                      // BNET_FAKE_CUDA=1: host-memory emulation for CPU-only tests
int device_count();
int current_device();             // -1 when unavailable
bool pointer_is_device(const void* p, int* dev_out);
// sysfs path of GPU `dev` ("/sys/devices/pci0000:16/…/0000:1b:00.0"), "" when unknown; `busid_out` gets "0000:1b:00.0"
std::string device_pci_path(int dev, std::string* busid_out = nullptr);
// device-side alias of pinned/registered host memory (nullptr when the GPU cannot read it directly)
void* host_device_alias(const void* host_ptr);

// ---- cross-process memory export / import (regMr for NCCL_PTR_CUDA) ----------
enum ExportKind : uint32_t { EXPORT_NONE = 0, EXPORT_CUDA_IPC = 1, EXPORT_POSIX_FD = 2, EXPORT_SAME_PROCESS = 3 };
struct MemExport {
  uint32_t kind;
  int32_t dev;
  uint64_t alloc_base;     // base VA of the whole allocation in the exporter
  uint64_t alloc_size;
  uint64_t pid;
  int32_t fd;              // EXPORT_POSIX_FD: fd number in the exporting process
  uint32_t pad;
  unsigned char ipc[64];   // EXPORT_CUDA_IPC: cudaIpcMemHandle_t
};
// Export the allocation that contains [ptr, ptr+size).  Returns 0 on success.
int export_memory(const void* ptr, size_t size, MemExport* out);
void release_export(MemExport* e);
// Map an exported allocation into this process for device `dev`; `fd` is a local
// fd (already transferred) for EXPORT_POSIX_FD.  Returns the local base VA.
int import_memory(const MemExport& e, int local_fd, int dev, void** base_out, void** cookie_out);
void release_import(const MemExport& e, void* base, void* cookie);

// ---- pinned host memory visible to the GPU -----------------------------------
int host_register(void* p, size_t n, void** dev_ptr_out);   // cudaHostRegister(mapped)
int host_unregister(void* p);
void* host_alloc_mapped(size_t n, void** dev_ptr_out);       // cudaHostAlloc(mapped|portable)
void host_free_mapped(void* p);

// ---- staged copies for the bounce paths ---------------------------------------
int memcpy_sync(void* dst, const void* src, size_t n, int dev);   // any direction, blocks
int enable_peer_access(int dev, int peer);

}  // namespace cuda
}  // namespace bnet

// Library-level entry points of libctr_b200.so: error text, version, device info, launch counter.
#include <stdarg.h>
#include <string.h>

#include <atomic>

#include "ctr_common.cuh"

namespace ctr {
static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}
}  // namespace ctr

extern "C" {
const char* ctr_last_error(void) { return ctr::g_err; }
int ctr_version(void) { return 1; }
int64_t ctr_kernel_launches(void) { return ctr::g_launches.load(); }

int ctr_enable_peer_access(int peer_device) {
  int dev = 0;
  CTR_CUDA(cudaGetDevice(&dev));
  if (peer_device == dev) return CTR_OK;
  int can = 0;
  CTR_CUDA(cudaDeviceCanAccessPeer(&can, dev, peer_device));
  if (!can) {
    ctr::set_error("ctr_enable_peer_access: device %d cannot access device %d over P2P", dev, peer_device);
    return CTR_ERR_UNSUPPORTED;
  }
  cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return CTR_OK; }
  if (e != cudaSuccess) {
    ctr::set_error("cudaDeviceEnablePeerAccess(%d) failed: %s", peer_device, cudaGetErrorString(e));
    return CTR_ERR_CUDA;
  }
  return CTR_OK;
}

// ---- peer-mappable buffers (row-sharded tables): plain cudaMalloc allocations exported / imported with CUDA IPC.
int ctr_peer_alloc(int64_t bytes, void** ptr) {
  CTR_REQUIRE(ptr != nullptr && bytes > 0, "ctr_peer_alloc: bad arguments");
  CTR_CUDA(cudaMalloc(ptr, (size_t)bytes));
  return CTR_OK;
}
int ctr_peer_free(void* ptr) {
  if (ptr) CTR_CUDA(cudaFree(ptr));
  return CTR_OK;
}
int ctr_ipc_export(void* ptr, unsigned char* handle64) {
  CTR_REQUIRE(ptr && handle64, "ctr_ipc_export: null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle is 64 bytes");
  cudaIpcMemHandle_t h;
  CTR_CUDA(cudaIpcGetMemHandle(&h, ptr));
  memcpy(handle64, &h, 64);
  return CTR_OK;
}
// Opens in the CURRENT device's context with lazy peer access: the mapping is usable by kernels of this device.
int ctr_ipc_import(const unsigned char* handle64, void** ptr) {
  CTR_REQUIRE(ptr && handle64, "ctr_ipc_import: null argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  CTR_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return CTR_OK;
}
int ctr_ipc_close(void* ptr) {
  if (ptr) CTR_CUDA(cudaIpcCloseMemHandle(ptr));
  return CTR_OK;
}

int ctr_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  CTR_CUDA(cudaGetDevice(&dev));
  int v = 0;
  if (sm_count) { CTR_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev)); *sm_count = v; }
  if (cc_major) { CTR_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, dev)); *cc_major = v; }
  if (cc_minor) { CTR_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, dev)); *cc_minor = v; }
  return CTR_OK;
}
}

// Shared helpers for the sm_90a CTR kernels: error reporting, launch accounting, warp primitives,
// cache-hinted 128-bit global accesses.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/ctr_b200.h"

namespace ctr {

void set_error(const char* fmt, ...);          // c_api.cu (thread-local message)
void count_launch(int n = 1);                  // c_api.cu
int sm_count();                                // cached multiprocessor count of the current device

#define CTR_REQUIRE(cond, ...)                                   \
  do {                                                           \
    if (!(cond)) {                                               \
      ctr::set_error(__VA_ARGS__);                               \
      return CTR_ERR_INVALID_ARG;                                \
    }                                                            \
  } while (0)

#define CTR_UNSUPPORTED(cond, ...)                               \
  do {                                                           \
    if (cond) {                                                  \
      ctr::set_error(__VA_ARGS__);                               \
      return CTR_ERR_UNSUPPORTED;                                \
    }                                                            \
  } while (0)

// Checks the launch (not the execution: kernels are asynchronous by contract).
#define CTR_CHECK_LAUNCH(name)                                                   \
  do {                                                                           \
    cudaError_t e__ = cudaGetLastError();                                        \
    if (e__ != cudaSuccess) {                                                    \
      ctr::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));    \
      return CTR_ERR_CUDA;                                                       \
    }                                                                            \
    ctr::count_launch();                                                         \
  } while (0)

#define CTR_CUDA(call)                                                           \
  do {                                                                           \
    cudaError_t e__ = (call);                                                    \
    if (e__ != cudaSuccess) {                                                    \
      ctr::set_error("%s failed: %s", #call, cudaGetErrorString(e__));           \
      return CTR_ERR_CUDA;                                                       \
    }                                                                            \
  } while (0)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// streaming (read-once) 128-bit load: read-only path, do not allocate in L1
__device__ __forceinline__ float4 ldg_stream_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
// write-once 128-bit store, evict-first in L2 (keeps hot table rows resident)
__device__ __forceinline__ void stg_stream_f4(float4* p, const float4& v) {
  asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ long long ldg_stream_i64(const long long* p) {
  long long r;
  asm volatile("ld.global.nc.L1::no_allocate.s64 %0, [%1];" : "=l"(r) : "l"(p));
  return r;
}

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }
static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace ctr

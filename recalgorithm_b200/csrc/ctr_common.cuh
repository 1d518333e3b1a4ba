// Shared helpers for the sm_90a CTR kernels: error reporting, launch accounting, warp primitives,
// cache-hinted 128-bit global accesses, and the host side of a launch (grid sizing, shared-memory attribute, launch
// check, compile-time shape dispatch).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <type_traits>

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
// 128-bit load through the L1 path.  The config-5 streams (the lookup backward's tile and d_tile rows, the gather's random
// 128-byte table rows) measured about 3 % faster this way than with ldg_stream_f4 (H100 SXM, 700 W).
__device__ __forceinline__ float4 ldg_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
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

// Grid of a launch that needs `need` CTAs, at most `cap` (grid-stride kernels: a few CTAs per SM fill the device).
static inline int capped_grid(long long need, long long cap) { return (int)(need < cap ? need : cap); }

// Launches k with `smem` bytes of dynamic shared memory (raising the kernel's limit past the default 48 KB when needed)
// and checks the launch; `what` names it in the error message.
template <class... P, class... A>
int launch(const char* what, void (*k)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, const A&... args) {
  if (smem > 48 * 1024) CTR_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k<<<grid, block, smem, st>>>(args...);
  CTR_CHECK_LAUNCH(what);
  return CTR_OK;
}

// Launches a persistent kernel k (its CTAs loop over the work) with one wave of resident CTAs: the occupancy of k at
// `block` threads and `smem` bytes times the SM count (one CTA per SM if the query fails, at most MAX_PER_SM per SM when
// given), capped at the `need` CTAs the work fills.  Raises the shared-memory limit first: the query depends on it.
template <int MAX_PER_SM = 0, class... P, class... A>
int launch_resident(const char* what, void (*k)(P...), long long need, int block, size_t smem, cudaStream_t st,
                    const A&... args) {
  if (smem > 48 * 1024) CTR_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, block, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  if (MAX_PER_SM > 0 && per_sm > MAX_PER_SM) per_sm = MAX_PER_SM;
  k<<<capped_grid(need, (long long)per_sm * sm_count()), block, smem, st>>>(args...);
  CTR_CHECK_LAUNCH(what);
  return CTR_OK;
}

// Compile-time dispatch: returns f(std::integral_constant<int, V>{}) for the V of Vs equal to v (the kernels take their
// shape class or method as a template argument).
template <int... Vs, class F>
int with_const(int v, F&& f) {
  int rc = CTR_OK;
  const bool hit = ((v == Vs && ((rc = f(std::integral_constant<int, Vs>{})), true)) || ...);
  if (!hit) {
    set_error("no kernel instantiation for %d", v);
    return CTR_ERR_INVALID_ARG;
  }
  return rc;
}
// The row kernels move a D-float row as LPR = D / 4 float4 lanes, for the power-of-two D in 4..128 their callers accept.
template <class F>
int with_lpr(int64_t D, F&& f) {
  return with_const<1, 2, 4, 8, 16, 32>((int)(D / 4), f);
}

}  // namespace ctr

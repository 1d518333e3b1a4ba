// wgmma / TMA / mbarrier PTX wrappers shared by the tensor-core kernels (sm_90a), the pipeline mechanics built on them
// (shared-memory alignment, the mbarrier ring, the producer / consumer role split, the 3xTF32 k-step, accumulation chains)
// and the host side of a tensor-core launch (workspace check, tensor-map encoding).
#pragma once
#include <cuda.h>

#include "ctr_common.cuh"

namespace ctr {
namespace tc {

constexpr int WG_M = 64;                 // rows of one warpgroup MMA (wgmma m64nNk8)
constexpr int KB = 32;                   // tf32 per 128-byte swizzle row
constexpr int NWG = 2;                   // consumer warpgroups per CTA
constexpr int NTHREADS = (NWG + 1) * 128;  // + one producer warpgroup (one TMA thread)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(bar), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// a warp-uniform copy of v (lets the compiler see that role branches never split a warpgroup)
__device__ __forceinline__ int warp_uniform(int v) { return __shfl_sync(0xffffffffu, v, 0); }
// register budget of the producer / consumer warpgroups (the producer only needs a handful)
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// barrier over the 128 threads of one warpgroup (ids 1.. ; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar)
      : "memory");
}

__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// a (4 values of one A fragment) -> hi = tf32(a), lo = tf32(a - hi)   (3xTF32: a.b ~= hi.bhi + lo.bhi + hi.blo)
__device__ __forceinline__ void tf32_split(const float (&a)[4], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float h = tf32_rna(a[q]);
    hi[q] = __float_as_uint(h);
    lo[q] = __float_as_uint(tf32_rna(a[q] - h));
  }
}

// GMMA shared-memory descriptor of a K-major operand with 8-row groups `8 * row_bytes` apart:
// row_bytes 128 = SWIZZLE_128B (layout 1), 64 = SWIZZLE_64B (2), 32 = SWIZZLE_32B (3).  Tiles are 1024-byte aligned.
// Advancing K by 8 tf32 (32 bytes) inside the swizzle span adds 2 to the descriptor.
__device__ __forceinline__ uint64_t gmma_desc_kmajor(uint32_t saddr, int row_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);                 // start address        bits [0,14)
  d |= (uint64_t)1 << 16;                                   // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)((8 * row_bytes) >> 4) << 32;              // stride byte offset   bits [32,46)
  d |= (uint64_t)(row_bytes == 128 ? 1 : row_bytes == 64 ? 2 : 3) << 62;
  return d;
}

// The A-fragment registers of a wgmma must not be rewritten before the wgmma.wait_group that retires it (ptxas only fences
// them, it does not wait).  Kernels therefore form every A fragment of a group up front and pass each one through this after
// the wait: the registers stay allocated to the group until then.
__device__ __forceinline__ void wgmma_keep(uint32_t (&r)[4]) {
  asm volatile("" : "+r"(r[0]), "+r"(r[1]), "+r"(r[2]), "+r"(r[3])::"memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] (+)= A[64 x 8] . B[8 x N], kind tf32, A from registers, B (N rows, K-major) from shared memory.
// A fragment of a thread (lane = 4 g + t of warp w of the warpgroup): a[0] = A[16w+g][t], a[1] = A[16w+g+8][t],
// a[2] = A[16w+g][t+4], a[3] = A[16w+g+8][t+4].  D fragment: d[4c+e] = D[16w+g][8c+2t+e], d[4c+2+e] = D[16w+g+8][8c+2t+e].
// scale_d == 0 overwrites D.
template <int N>
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t bdesc, int scale_d);
template <>
__device__ __forceinline__ void wgmma_tf32_rs<32>(float (&d)[16], const uint32_t (&a)[4], uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_tf32_rs<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_tf32_rs<96>(float (&d)[48], const uint32_t (&a)[4], uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %53, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, {%48,%49,%50,%51}, %52, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_tf32_rs<128>(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d));
}

// One 3xTF32 k-step, D (+)= (ah + al) . (bhi + blo), with B `off` descriptor units into its hi and lo tiles: the small terms
// first, the dominant hi.hi term last.  scale_d == 0 starts a new accumulation chain.
template <int N>
__device__ __forceinline__ void mma_3xtf32(float (&d)[N / 2], const uint32_t (&ah)[4], const uint32_t (&al)[4], uint64_t bhi,
                                           uint64_t blo, uint64_t off, int scale_d) {
  wgmma_tf32_rs<N>(d, al, bhi + off, scale_d);
  wgmma_tf32_rs<N>(d, ah, blo + off, 1);
  wgmma_tf32_rs<N>(d, ah, bhi + off, 1);
}
// Waits for every committed wgmma group, then releases the A fragments (hi, lo) those groups read.
template <int NK>
__device__ __forceinline__ void wgmma_wait_keep(uint32_t (&ah)[NK][4], uint32_t (&al)[NK][4]) {
  wgmma_wait<0>();
#pragma unroll
  for (int k = 0; k < NK; ++k) { wgmma_keep(ah[k]); wgmma_keep(al[k]); }
}

// Accumulation chains: the tensor core adds each K=8 product group into the fp32 accumulator with truncation, so a long
// chain drifts by ~0.5 ulp per MMA.  Kernels therefore accumulate `len` steps from zero into dacc and then add dacc into
// acc (round-to-nearest).  Step i of n: the first of a chain overwrites dacc (scale_d 0), the last one drains it.
__device__ __forceinline__ bool chain_first(int i, int len) { return i % len == 0; }
__device__ __forceinline__ bool chain_last(int i, int n, int len) { return (i + 1) % len == 0 || i + 1 == n; }
template <int N>
__device__ __forceinline__ void chain_drain(float (&acc)[N], const float (&dacc)[N]) {
#pragma unroll
  for (int q = 0; q < N; ++q) acc[q] += dacc[q];
}

// 3xTF32 operand in memory: dst[idx] = tf32(v) (the hi copy), dst[total + idx] = v - tf32(v) (the lo copy)
__device__ __forceinline__ void store_split(float* dst, size_t total, size_t idx, float v) {
  const float hi = tf32_rna(v);
  dst[idx] = hi;
  dst[total + idx] = v - hi;
}

// SWIZZLE_128B tiles must be 1024-byte aligned: the kernels align their dynamic shared memory here, and every launch
// asks for 1 KB of slack on top of the layout.
__device__ __forceinline__ uint8_t* align_1024(uint8_t* smem_raw) {
  return smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
}

// The ring of SB shared-memory stages between the TMA producer thread and the 4 NWG consumer warps.  Stage s has a `full`
// barrier (one arrival + the bytes of its TMA loads) and an `empty` barrier (one arrival per consumer warp); bar0 points
// at 2 SB 8-byte barriers.  The producer and every consumer thread walk the stages in the same order, each with its own
// copy of the (stage, phase) position.
struct Ring {
  uint32_t bar0;
  int nstages;
  int s = 0;
  uint32_t ph = 0;

  __device__ __forceinline__ Ring(uint32_t bar0_, int nstages_) : bar0(bar0_), nstages(nstages_) {}
  __device__ __forceinline__ uint32_t full() const { return bar0 + 8 * s; }
  __device__ __forceinline__ uint32_t empty() const { return bar0 + 8 * (nstages + s); }
  __device__ __forceinline__ void advance() {
    if (++s == nstages) { s = 0; ph ^= 1; }
  }
  // every thread of the CTA: thread 0 initialises the barriers, all return once they are visible
  __device__ __forceinline__ void init() const {
    if (threadIdx.x == 0) {
      for (int i = 0; i < nstages; ++i) { mbar_init(bar0 + 8 * i, 1); mbar_init(bar0 + 8 * (nstages + i), NWG * 4); }
      fence_barrier_init();
    }
    __syncthreads();
  }
  struct Slot {
    int stage;
    uint32_t full;      // the barrier the stage's TMA loads complete on
  };
  // producer: waits until the next stage is free and arms it for `bytes`
  __device__ __forceinline__ Slot acquire(uint32_t bytes) {
    mbar_wait(empty(), ph ^ 1);
    mbar_expect_tx(full(), bytes);
    const Slot slot = {s, full()};
    advance();
    return slot;
  }
  // consumer: waits until the current stage has landed and returns its index
  __device__ __forceinline__ int wait() const {
    mbar_wait(full(), ph);
    return s;
  }
  // consumer warp: done with the current stage (after the wgmma.wait that covers it)
  __device__ __forceinline__ void release(int lane) {
    if (lane == 0) mbar_arrive(empty());
    advance();
  }
};

// Role split of a CTA of NTHREADS: the producer warpgroup drops to 40 registers per thread and its first thread runs
// `producer`; the consumer warpgroups (warps 0 .. 4 NWG - 1) get 232.  Returns true on the producer warpgroup, which then
// has nothing left to do.
template <class Producer>
__device__ __forceinline__ bool producer_role(int warp, int lane, Producer&& producer) {
  if (warp >= NWG * 4) {
    setmaxnreg_dec<40>();
    if (warp == NWG * 4 && lane == 0) producer();
    return true;
  }
  setmaxnreg_inc<232>();
  return false;
}

// ------------------------------------------------------------------------------------------------ host
static inline int64_t pad_to(int64_t v, int64_t q) { return (v + q - 1) / q * q; }
// wgmma N (or K) class of a width v <= 128: 32, 64 or 128
static inline int pad3(int64_t v) { return v <= 32 ? 32 : v <= 64 ? 64 : 128; }
// The caller's workspace: at least `need` bytes (size_fn tells how many), 128-byte aligned.
static inline int check_workspace(const char* fn, const char* size_fn, const void* ws, int64_t bytes, int64_t need) {
  CTR_REQUIRE(ws != nullptr && bytes >= need, "%s: workspace of %lld bytes required (%s), got %lld", fn, (long long)need,
              size_fn, (long long)bytes);
  CTR_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 127) == 0, "%s: workspace must be 128-byte aligned", fn);
  return CTR_OK;
}

// Tensor map of a float32 tensor at `base`: dims and box innermost first, byte_strides of dimensions 1 .. rank - 1.
static inline int encode_tmap(const char* fn, CUtensorMap* map, int rank, const void* base, const cuuint64_t* dims,
                              const cuuint64_t* byte_strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle) {
  typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeTiledFn enc = nullptr;
  if (enc == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      enc = reinterpret_cast<EncodeTiledFn>(p);
  }
  if (enc == nullptr) {
    set_error("%s: cuTensorMapEncodeTiled is not available from the driver", fn);
    return CTR_ERR_CUDA;
  }
  const cuuint32_t elem_strides[5] = {1, 1, 1, 1, 1};
  CUresult cr = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, const_cast<void*>(base), dims, byte_strides, box,
                    elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    set_error("%s: cuTensorMapEncodeTiled failed with CUresult %d", fn, (int)cr);
    return CTR_ERR_CUDA;
  }
  return CTR_OK;
}

}  // namespace tc
}  // namespace ctr

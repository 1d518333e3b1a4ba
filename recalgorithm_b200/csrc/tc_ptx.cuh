// wgmma / TMA / mbarrier PTX wrappers shared by the tensor-core kernels (sm_90a), the pipeline mechanics built on them
// (shared-memory alignment, the mbarrier ring, the producer / consumer role split, the 3xTF32 k-step, accumulation chains,
// the consumer loop of the batch-reduction weight-gradient GEMMs, the one weight-gradient kernel of the dense layers built
// on it, the row-chunk and K-sliced row GEMMs of the dense-layer kernels and the cross-network epilogue) and the host side of a tensor-core launch (workspace check,
// tensor-map encoding, batch slices, ring depth and launch of the weight-gradient kernels).
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
// barrier over the 256 threads of both consumer warpgroups (id 1: kernels that use it do not use wg_bar_sync)
__device__ __forceinline__ void consumers_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
// makes this thread's generic-proxy shared-memory writes visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

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
// store_split into a K-major SWIZZLE_128B B-operand tile written by threads instead of TMA: `rows` 128-byte rows of 32 tf32
// (hi tile, then the lo tile rows * 128 bytes on), 1024-byte aligned.  Element (k, b) sits at byte k * 128 + 4 b with its
// 16-byte chunk index XORed with k & 7, the placement TMA's SWIZZLE_128B gives and gmma_desc_kmajor(.., 128) reads.
__device__ __forceinline__ void store_split_sw128(float* tile, int rows, int k, int b, float v) {
  const uint32_t o = (uint32_t)(k * 128 + b * 4);
  store_split(tile, rows * 32, (o ^ (((o >> 7) & 7u) << 4)) / 4, v);
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

// Batch slice `slice` of `nslices` over n_units (chunks or samples) of a batch-reduction grid: [beg, end), up to
// ceil(n_units / nslices) units; empty for the slices past the end.
__device__ __forceinline__ void batch_slice(int slice, int nslices, int n_units, int& beg, int& end) {
  const int per_slice = (n_units + nslices - 1) / nslices;
  beg = min(n_units, slice * per_slice);
  end = min(n_units, beg + per_slice);
}

// Batch-reduction GEMM of the weight-gradient kernels: acc[DW_NC rows][N] = sum_b P[b, row] Q[b, k] over the chunks
// [c_beg, c_end) of DW_BC samples, b < B.  A = P^T (rows x samples) from a TMA-staged P chunk, B = Q^T (N x samples)
// generated on chip.
constexpr int DW_BC = KB;                    // samples per chunk: the K of 4 k-steps, one 128-byte swizzle row of Q^T
constexpr int DW_NC = NWG * WG_M;            // rows (P columns) per CTA

// The consumer side, run by all 256 consumer threads, one ring stage per chunk.  The stage's Q^T tiles sit at
// qts + stage * 2 N 128 (written here); its P chunk is wherever the producer put it.  Per chunk b0 = c DW_BC:
//   stage_chunk(b0)   the caller's per-chunk staging for q_of (it may use consumers_bar), or nothing;
//   Q^T (hi | lo) into the stage's swizzled tiles, element (k, b) = q_of(k, b0, b) for b0 + b < B, else 0;
//   A fragments of P^T, element (row, b) = p_of(stage, b, row): row = this thread's nl0 or nl0 + 8, b < DW_BC;
//   4 3xTF32 k-steps, then the stage is released; chains of 8 chunks (32 k-steps, 96 MMAs) drained into acc.
// The caller owns the shared-memory layout, the producer and the epilogue (acc: the D fragment of rows nl0, nl0 + 8).
template <int N, class Stage, class QOf, class POf>
__device__ __forceinline__ void batch_reduce(float (&acc)[N / 2], Ring& ring, uint8_t* qts, int c_beg, int c_end, int B,
                                             int lane, int nl0, Stage&& stage_chunk, QOf&& q_of, POf&& p_of) {
  constexpr int qt_bytes = 2 * N * 128;
  constexpr int CHAIN = 8;                   // chunks per accumulation chain
  const int t = lane & 3;
  float dacc[N / 2];
#pragma unroll
  for (int q = 0; q < N / 2; ++q) { acc[q] = 0.f; dacc[q] = 0.f; }
  for (int c = c_beg; c < c_end; ++c) {
    const int b0 = c * DW_BC;
    stage_chunk(b0);
    const int s = ring.wait();
    float* qt = reinterpret_cast<float*>(qts + s * qt_bytes);
    for (int idx = threadIdx.x; idx < N * DW_BC; idx += NWG * 128) {
      const int k = idx / DW_BC, b = idx % DW_BC;
      store_split_sw128(qt, N, k, b, b0 + b < B ? q_of(k, b0, b) : 0.f);
    }
    fence_proxy_async();
    consumers_bar();
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      float a[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) a[q] = p_of(s, 8 * ks + t + 4 * (q >> 1), nl0 + 8 * (q & 1));
      tf32_split(a, ah[ks], al[ks]);
    }
    const bool chain_start = chain_first(c - c_beg, CHAIN);
    const uint64_t bhi = gmma_desc_kmajor(smem_u32(qt), 128);
    const uint64_t blo = gmma_desc_kmajor(smem_u32(qt + N * 32), 128);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) mma_3xtf32<N>(dacc, ah[ks], al[ks], bhi, blo, 2 * ks, (chain_start && ks == 0) ? 0 : 1);
    wgmma_commit();
    wgmma_wait_keep(ah, al);
    ring.release(lane);
    if (chain_last(c - c_beg, c_end - c_beg, CHAIN)) chain_drain(acc, dacc);
  }
}

// The weight-gradient kernel of the dense layers (residual unit, MMoE, PLE, AutoInt) around batch_reduce: result row n,
// input k0 + k = sum over b < rows_total of P[b, n] Q[b, k0 + k].  P is a [rows_total x units] workspace tensor streamed by
// TMA in [DW_BC samples x DW_NC units] chunks (no swizzle); Q is q (rows_total, d), or q [qmask > 0] with Rows::mask_q.
// CTA (x, y) owns the DW_NC units x % ngroups, the batch slice x / ngroups of nslices and the N inputs from k0 = y N, and
// adds its partial result with one atomic per element into rows.row(n).  Each layer's Rows type, small and trivially
// copyable, gives `GradRow row(int n) const` and three compile-time flags: row_sums (also sum each row over the samples
// into its bias; the y = 0 CTAs only), mask_q, and slice_d (the grid's y dimension slices the inputs; without it k0 = 0).
// Being compile-time, they cost the layers that do not use them nothing in the per-element loops: a run-time k0, for one,
// is rematerialised from blockIdx.y for every element at this register budget.
struct GradRow {
  float* dst = nullptr;                      // element k of the row at dst[k * stride]; null for padding rows
  int stride = 0;
  float* bias = nullptr;                     // the row's batch sum (Rows::row_sums), or null
};

// atomicAdd(p, v) with the result unused, p in global memory: the compiler cannot always tell that a pointer taken from a
// Rows value is global, and a generic atomic tests every address for the shared window first.
__device__ __forceinline__ void red_add_global(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(__cvta_generic_to_global(p)), "f"(v) : "memory");
}

// shared memory of weight_grad_wgmma_kernel: per stage the Q^T tiles, one P chunk and the two ring barriers
__host__ __device__ constexpr int dw_smem_bytes(int N, int SB) { return SB * (2 * N * 128 + DW_BC * DW_NC * 4 + 16); }

template <int N, class Rows>
__global__ void __launch_bounds__(NTHREADS, 1)
weight_grad_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_p, const float* __restrict__ q,
                         const float* __restrict__ qmask, const Rows rows, int rows_total, int d, int ngroups, int nslices,
                         int SB) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int qt_bytes = 2 * N * 128;                     // Q^T tiles [N x 32 samples] (hi | lo), 128B-swizzled
  constexpr int p_floats = DW_BC * DW_NC;                   // one P chunk [32 samples x 128 units]
  uint8_t* qts = smem;
  float* ps = reinterpret_cast<float*>(smem + SB * qt_bytes);
  Ring ring(smem_u32(ps + SB * p_floats), SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int group = blockIdx.x % ngroups, k0 = Rows::slice_d ? blockIdx.y * N : 0;
  int c_beg, c_end;
  batch_slice(blockIdx.x / ngroups, nslices, (rows_total + DW_BC - 1) / DW_BC, c_beg, c_end);
  const int n0 = group * DW_NC;

  ring.init();
  // ============================ TMA producer: P chunks [32 samples x 128 units] ============================
  if (producer_role(warp, lane, [&] {
        for (int c = c_beg; c < c_end; ++c) {
          const Ring::Slot slot = ring.acquire(p_floats * 4);
          tma_load_2d(smem_u32(ps + (size_t)slot.stage * p_floats), &tmap_p, n0, c * DW_BC, slot.full);
        }
      }))
    return;

  // ============================ consumers: B = Q^T generated on chip, A = P^T ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3;
  float rsum[2] = {0.f, 0.f};                               // Rows::row_sums: sum_b of this thread's two rows
  const int nl0 = wg * WG_M + w * 16 + g;                   // this thread's A rows: units n0 + nl0 (+8)
  float acc[N / 2];
  batch_reduce<N>(
      acc, ring, qts, c_beg, c_end, rows_total, lane, nl0, [](int) {},
      [&](int k, int b0, int b) {
        if (k0 + k >= d) return 0.f;
        const size_t o = (size_t)(b0 + b) * d + k0 + k;
        return (!Rows::mask_q || __ldg(qmask + o) > 0.f) ? __ldg(q + o) : 0.f;
      },
      [&](int s, int b, int nl) {
        const float v = ps[(size_t)s * p_floats + b * DW_NC + nl];
        if (Rows::row_sums) rsum[nl == nl0 ? 0 : 1] += v;
        return v;
      });
  if (c_end <= c_beg) return;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const GradRow row = rows.row(n0 + nl0 + 8 * r);
#pragma unroll
    for (int cc = 0; cc < N / 8; ++cc) {
#pragma unroll
      for (int x = 0; x < 2; ++x) {
        const int k = k0 + 8 * cc + 2 * t + x;
        if (row.dst != nullptr && k < d) red_add_global(row.dst + (size_t)k * row.stride, acc[4 * cc + 2 * r + x]);
      }
    }
    if (Rows::row_sums) {
      float v = rsum[r];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      if (blockIdx.y == 0 && t == 0 && row.bias != nullptr) red_add_global(row.bias, v);
    }
  }
}

// Row-chunk GEMMs of the dense-layer kernels (residual unit, MMoE): 64 staged rows of an input of width DP (32 / 64 / 96 /
// 128) times a chunk of HC hidden units, whose result stays in registers and feeds the next GEMM as A fragments.
//   rows operand    [HC units x DP] K-major, streamed from a [2 R][DP] map (hi copy, then the lo copy R rows on);
//   hidden operand  [DP x HC units] K-major, streamed from a [2 DP][R] map whose units are in perm8 order.
namespace rows {

constexpr int HC = 32;                       // hidden units per chunk: N of the row GEMMs, K of the hidden GEMMs
constexpr int CHAIN = 32 / (HC / 8);         // hidden chunks per accumulation chain: 32 k-steps x 3 = 96 MMAs

// The wgmma accumulator gives thread (g, t) columns 8c + 2t and 8c + 2t + 1 of each 8-column group c, and the A fragment of
// k-step c wants columns 8c + t and 8c + t + 4.  Since a sum over k does not depend on its order, the fragment takes the
// accumulator's two columns as its k = t and k = t + 4, and the hidden operand holds its units permuted within each group of
// 8 to match: unit held at k position `k` is, within its group of 8, 2m for k = m < 4 and 2(m - 4) + 1 for k = m >= 4.
__host__ __device__ __forceinline__ int perm8(int k) {
  const int m = k & 7;
  return (k & ~7) | (m < 4 ? 2 * m : 2 * m - 7);
}

__host__ __device__ constexpr int row_pitch(int DP) { return DP + 4; }   // staged rows: conflict-free A-fragment reads
__host__ __device__ constexpr int stage_bytes(int DP) { return 2 * HC * DP * 4; }

// TMA loads of chunk j (units j HC ..) into a stage (hi tile, then lo tile): a rows operand is DP / 32 boxes of [HC x 32]
// per copy from a map of 2 R rows; a hidden operand one box of [DP x 32] per copy.
template <int DP>
__device__ __forceinline__ void load_rows_operand(uint32_t dst, const CUtensorMap* map, int j, int R, uint32_t bar) {
#pragma unroll
  for (int kb = 0; kb < DP / KB; ++kb) {
    tma_load_2d(dst + kb * HC * 128, map, kb * KB, j * HC, bar);
    tma_load_2d(dst + HC * DP * 4 + kb * HC * 128, map, kb * KB, R + j * HC, bar);
  }
}
template <int DP>
__device__ __forceinline__ void load_hidden_operand(uint32_t dst, const CUtensorMap* map, int j, uint32_t bar) {
  tma_load_2d(dst, map, j * HC, 0, bar);
  tma_load_2d(dst + DP * 128, map, j * HC, DP, bar);
}

// D[64 x HC] = R[64 x DP] . B: R = this warpgroup's 64 staged rows (pitch row_pitch(DP)), B = a rows-operand stage.
// Issued one 32-column block (4 k-steps) at a time, so that only 32 fragment registers are live.
template <int DP>
__device__ __forceinline__ void gemm_rows(float (&d)[HC / 2], const float* rows, int r0, int t, uint32_t stage) {
  constexpr int LD = row_pitch(DP);
  const uint64_t bhi = gmma_desc_kmajor(stage, 128);
  const uint64_t blo = gmma_desc_kmajor(stage + HC * DP * 4, 128);
#pragma unroll
  for (int kb = 0; kb < DP / KB; ++kb) {
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      float a[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) a[q] = rows[(r0 + 8 * (q & 1)) * LD + kb * KB + 8 * ks + t + 4 * (q >> 1)];
      tf32_split(a, ah[ks], al[ks]);
    }
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      mma_3xtf32<HC>(d, ah[ks], al[ks], bhi, blo, (uint64_t)(kb * (HC * 128 / 16) + 2 * ks), (kb | ks) ? 1 : 0);
    wgmma_commit();
    wgmma_wait_keep(ah, al);
  }
}

// A fragments of a hidden chunk held in accumulator layout: k-step c takes the thread's columns 8c + 2t (as k = t) and
// 8c + 2t + 1 (as k = t + 4) of rows g and g + 8 -- the order perm8 gives the B operand.
__device__ __forceinline__ void acc_to_a(const float (&v)[HC / 2], uint32_t (&hh)[HC / 8][4], uint32_t (&hl)[HC / 8][4]) {
#pragma unroll
  for (int c = 0; c < HC / 8; ++c) {
    const float a[4] = {v[4 * c], v[4 * c + 2], v[4 * c + 1], v[4 * c + 3]};
    tf32_split(a, hh[c], hl[c]);
  }
}

// D[64 x DP] (+)= Hc[64 x HC] . B: Hc from acc_to_a, B = a hidden-operand stage; `start` begins a new chain.
template <int DP>
__device__ __forceinline__ void gemm_hidden(float (&d)[DP / 2], uint32_t (&hh)[HC / 8][4], uint32_t (&hl)[HC / 8][4],
                                            uint32_t stage, bool start) {
  const uint64_t bhi = gmma_desc_kmajor(stage, 128);
  const uint64_t blo = gmma_desc_kmajor(stage + DP * 128, 128);
  wgmma_fence();
#pragma unroll
  for (int c = 0; c < HC / 8; ++c) mma_3xtf32<DP>(d, hh[c], hl[c], bhi, blo, (uint64_t)(2 * c), (start && c == 0) ? 0 : 1);
  wgmma_commit();
  wgmma_wait_keep(hh, hl);
}

// Stages this warpgroup's 64 rows of a (B, d) tensor, zero padded to DP columns and past B, with ordinary loads (the rows
// need not be 16-byte aligned); with `mask`, the rows of src [mask > 0] instead.
template <int DP>
__device__ __forceinline__ void stage_rows(float* dst, const float* __restrict__ src, const float* __restrict__ mask,
                                           long long base, int B, int d, int tw) {
  constexpr int LD = row_pitch(DP);
  for (int idx = tw; idx < WG_M * DP; idx += 128) {
    const int r = idx / DP, c = idx % DP;
    float v = 0.f;
    if (c < d && base + r < B) {
      const size_t o = (size_t)(base + r) * d + c;
      v = (mask == nullptr || __ldg(mask + o) > 0.f) ? __ldg(src + o) : 0.f;
    }
    dst[r * LD + c] = v;
  }
}

// K-sliced row GEMMs over inputs up to 512 wide (PLE, DCN-V2): both warpgroups read the same staged rows, and a ring stage
// holds [2 NW units x 32 inputs] (hi tile, then lo tile), of which warpgroup wg takes units wg NW .. wg NW + NW - 1.  The
// ring depth does not depend on the input width.
template <int NW>
__host__ __device__ constexpr int ks_stage_bytes() { return 2 * 2 * NW * KB * 4; }

// TMA loads of one stage: units u0 .. u0 + 2 NW - 1, inputs 32 kb .., hi then lo, from a [2 NP][KP] map (boxes of
// [2 NW x 32]; the lo copy starts NP rows on).
template <int NW>
__device__ __forceinline__ void load_ks_stage(uint32_t dst, const CUtensorMap* map, int u0, int kb, int NP, uint32_t bar) {
  tma_load_2d(dst, map, kb * KB, u0, bar);
  tma_load_2d(dst + 2 * NW * 128, map, kb * KB, NP + u0, bar);
}

// D[64 x NW] = X[64 x 32 nk] . B over the next nk ring stages: X = the tile's staged rows (pitch ldx), B = this warpgroup's
// NW-unit half of each stage.  One 32-input slice (4 k-steps) per stage, each drained into d on its own: the tensor core
// truncates as it accumulates, and with 96-MMA chains PLE's widest inputs missed the fp32 bars by up to 1.2x (the softmax
// turns a gate logit's absolute error into the gate's relative error).
template <int NW>
__device__ __forceinline__ void gemm_ks(float (&d)[NW / 2], const float* xs, int ldx, int nk, int r0, int t, int lane,
                                        int wg, Ring& ring, uint32_t sbase) {
  float dacc[NW / 2];
#pragma unroll
  for (int q = 0; q < NW / 2; ++q) { d[q] = 0.f; dacc[q] = 0.f; }
  for (int kb = 0; kb < nk; ++kb) {
    const uint32_t st = sbase + ring.wait() * ks_stage_bytes<NW>() + wg * NW * 128;
    const uint64_t bhi = gmma_desc_kmajor(st, 128), blo = gmma_desc_kmajor(st + 2 * NW * 128, 128);
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      float a[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) a[q] = xs[(r0 + 8 * (q & 1)) * ldx + kb * KB + 8 * ks + t + 4 * (q >> 1)];
      tf32_split(a, ah[ks], al[ks]);
    }
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) mma_3xtf32<NW>(dacc, ah[ks], al[ks], bhi, blo, (uint64_t)(2 * ks), ks == 0 ? 0 : 1);
    wgmma_commit();
    wgmma_wait_keep(ah, al);
    ring.release(lane);
    chain_drain(d, dacc);
  }
}

// The epilogue of a cross-network K-sliced row GEMM slice (DCN-V2, DCN-Mix) for this thread's gemm_ks<NW> accumulator
// (rows r0, r0 + 8 of the 64-sample tile at `base`, columns c0 + 8 c + e).  The layer's Args type names the fields read here:
//   EPI_STORE  y (B, ldy) = acc;
//   EPI_FWD    z = acc + bias, x_{l+1} = x0 o z + xl into y, z into z_out (or not);
//   EPI_BWD    dx_l = g + acc into y (or nothing), dx0 (+)= g o z (+ dx_l with dx0_add_dx).
// Every operand is loaded before the first store: the pointers may alias, so a load would otherwise wait for each store
// before it, one memory latency per element.
enum CrossEpilogue { EPI_STORE = 0, EPI_FWD = 1, EPI_BWD = 2 };
template <int NW, class Args>
__device__ __forceinline__ void cross_epilogue(const Args& p, const float (&acc)[NW / 2], long long base, int r0, int c0) {
  if (p.epi == EPI_STORE) {
#pragma unroll
    for (int k = 0; k < NW / 2; ++k) {
      const int col = c0 + 8 * (k >> 2) + (k & 1);
      const long long row = base + r0 + 8 * ((k >> 1) & 1);
      if (row < p.B && col < p.ldy) p.y[(size_t)row * p.ldy + col] = acc[k];
    }
    return;
  }
  const bool fwd = p.epi == EPI_FWD;
  float u0[NW / 2], u1[NW / 2], u2[NW / 2];  // FWD: x0, x_l, b;  BWD: g, z, the old dx0
#pragma unroll
  for (int k = 0; k < NW / 2; ++k) {
    const int col = c0 + 8 * (k >> 2) + (k & 1);
    const long long row = base + r0 + 8 * ((k >> 1) & 1);
    u0[k] = u1[k] = u2[k] = 0.f;
    if (row < p.B && col < p.d) {
      const size_t o = (size_t)row * p.d + col;
      u0[k] = fwd ? p.x0[o] : p.g[o];
      u1[k] = fwd ? p.xl[o] : p.z[o];
      u2[k] = fwd ? __ldg(p.bias + col) : p.dx0_accumulate ? p.dx0[o] : 0.f;
    }
  }
#pragma unroll
  for (int k = 0; k < NW / 2; ++k) {
    const int col = c0 + 8 * (k >> 2) + (k & 1);
    const long long row = base + r0 + 8 * ((k >> 1) & 1);
    if (row >= p.B || col >= p.d) continue;
    const size_t o = (size_t)row * p.d + col;
    if (fwd) {
      const float z = acc[k] + u2[k];
      if (p.z_out != nullptr) p.z_out[o] = z;
      p.y[o] = u0[k] * z + u1[k];
    } else {
      const float dx = u0[k] + acc[k];
      float d0 = u0[k] * u1[k];
      if (p.dx0_add_dx) d0 += dx;
      else if (p.y != nullptr) p.y[o] = dx;
      p.dx0[o] = p.dx0_accumulate ? u2[k] + d0 : d0;
    }
  }
}

}  // namespace rows

// ------------------------------------------------------------------------------------------------ host
constexpr size_t SMEM_CAP = 226 * 1024;     // dynamic shared memory per CTA on sm_90 (227 KB) less slack

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

// a row-major [outer x inner] float matrix, one box of [box_outer x box_inner]
static inline int encode_2d(const char* fn, CUtensorMap* map, const void* base, uint64_t inner, uint64_t outer,
                            uint32_t box_inner, uint32_t box_outer, CUtensorMapSwizzle sw) {
  const cuuint64_t gdim[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  const cuuint64_t gstr[1] = {(cuuint64_t)inner * sizeof(float)};
  const cuuint32_t box[2] = {box_inner, box_outer};
  return encode_tmap(fn, map, 2, base, gdim, gstr, box, sw);
}

// Slices per group of a batch-reduction grid of ngroups x nslices CTAs: one wave over the SMs, at most one per unit.
static inline int batch_slices(int sms, int64_t ngroups, int64_t n_units) {
  int64_t n = sms / ngroups;
  if (n < 1) n = 1;
  return (int)(n < n_units ? n : n_units);
}
// Ring stages of a batch-reduction kernel: as many as fit in SMEM_CAP next to `fixed` bytes (slack included), at most 4.
static inline int stages_that_fit(size_t fixed, size_t stage) {
  const size_t sb = (SMEM_CAP - fixed) / stage;
  return (int)(sb < 4 ? sb : 4);
}
// Launches weight_grad_wgmma_kernel<N, Rows> over P = p (rows_total rows of `units` floats) and Q = q (rows_total rows of
// d floats, masked by qmask with Rows::mask_q) for n_ds slices of N inputs: the batch slices of each input slice share
// one wave over the SMs (n_ds > 1 needs Rows::slice_d); `what` names the launch in error messages, `fn` the entry.
template <int N, class Rows>
static inline int launch_weight_grad(const char* fn, const char* what, const Rows& rows, const float* p, int64_t units,
                                     int64_t rows_total, const float* q, const float* qmask, int d, int n_ds,
                                     cudaStream_t st) {
  CUtensorMap map;
  if (int rc = encode_2d(fn, &map, p, units, rows_total, DW_NC, DW_BC, CU_TENSOR_MAP_SWIZZLE_NONE)) return rc;
  const int ngroups = (int)((units + DW_NC - 1) / DW_NC);
  const int nslices = batch_slices(sm_count() / n_ds, ngroups, (rows_total + DW_BC - 1) / DW_BC);
  const int sb = stages_that_fit(1024, dw_smem_bytes(N, 1));
  return launch(what, weight_grad_wgmma_kernel<N, Rows>, dim3(ngroups * nslices, n_ds), NTHREADS, dw_smem_bytes(N, sb) + 1024,
                st, map, q, qmask, rows, (int)rows_total, d, ngroups, nslices, sb);
}

namespace rows {
// Maps of the prepped operands at `base` (hi copy, then lo copy): rows operand [2 R][DP], boxes of [HC x 32]; hidden
// operand [2 DP][R], boxes of [DP x 32].
static inline int encode_rows_operand(const char* fn, CUtensorMap* map, const float* base, int DP, int64_t R) {
  return encode_2d(fn, map, base, DP, 2 * R, KB, HC, CU_TENSOR_MAP_SWIZZLE_128B);
}
static inline int encode_hidden_operand(const char* fn, CUtensorMap* map, const float* base, int DP, int64_t R) {
  return encode_2d(fn, map, base, R, 2 * DP, KB, DP, CU_TENSOR_MAP_SWIZZLE_128B);
}
// input width class of the row GEMMs: d rounded up to 32, 64, 96 or 128
static inline int dp_class(int64_t d) { return d <= 32 ? 32 : d <= 64 ? 64 : d <= 96 ? 96 : 128; }
}  // namespace rows

}  // namespace tc
}  // namespace ctr

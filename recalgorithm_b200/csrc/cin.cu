// Row CIN (SURVEY.md section 8a): the xDeepFM compressed-interaction layer.
//
// Reference: cin_layer(x0, xk, hk_1, index) -- xDeepFM/cin_layer.py:17-30
//   outer[b,d,i,j] = xk[b,i,d] * x0[b,j,d]; reshape (B, D, hk*m) with flat index i*m+j; conv1d with a
//   (1, hk*m, hk_1) filter == matmul over the last axis; transpose -> (B, hk_1, D).  The reference
//   materialises the (B, D, hk*m) outer tensor (2 GB at BASELINE config 3, layer 2).
//
// H100 mapping -- the one genuinely dense contraction of the hot path, so it runs on the tensor cores (wgmma):
//   GEMM view  C[M x N] = A[M x K] . B[K x N],  M = B*D rows r = (b,d),  K = hk*m,  N = hk_1.
//   * A (the outer product) is never written anywhere: it is formed in registers, directly in the wgmma A-fragment
//     layout.  Each thread of a consumer warpgroup owns two rows r of the 64-row warpgroup tile, keeps the x0 values of
//     its fragment columns in registers and, for every K-block i, multiplies them by xk[b,i,d]
//     (K is re-ordered as i*32 + j, zero padded from m to 32, so one K-block == one i == one 128-byte swizzle row);
//   * B (the filter) is pre-transposed/padded once per call into that K order (workspace) and streamed by TMA
//     (cp.async.bulk.tensor, SWIZZLE_128B) through an mbarrier pipeline shared by the CTA's two consumer warpgroups;
//   * wgmma.mma_async m64nNk8 kind tf32 (A from registers, B from shared memory, N = hk_1 padded to 32/64/128),
//     fp32 accumulators in registers;
//   * fp32-class accuracy (north_star: 1e-5) comes from the 3xTF32 split  A.B ~= Ahi.Bhi + Alo.Bhi + Ahi.Blo
//     with fp32 accumulation (error ~2^-22 per product); precision=1 runs a single TF32 pass (~1e-3);
//   * epilogue: accumulators -> shared memory -> (B, hk_1, D) stores + the pooled sum over D.
//   Shapes outside the tensor path's limits (m > 32, hk_1 > 128, D not a power of two <= 32) use a plain
//   CUDA-core kernel.  The backward pass is in cin_bwd.cu.
#include <stdlib.h>

#include "tc_ptx.cuh"

namespace ctr {
namespace cin {
using namespace ctr::tc;

// one K-block == KB tf32 == one i (128 B == swizzle span)
constexpr int TILE_M = NWG * WG_M;        // rows per CTA tile
constexpr int EPI_LD = WG_M + 4;          // row stride (floats) of the epilogue staging: conflict-free fragment stores

__host__ __device__ inline int fwd_smem_bytes(int N, int passes, int stages) {
  return stages * (passes == 3 ? 2 : 1) * N * 128 + NWG * N * EPI_LD * 4 + 8 * 2 * stages;
}

// ------------------------------------------------------------------------------------------------ kernels
// filter (hk*m, H) -> Wt[2][NP][KP]: [0] = tf32-rounded value, [1] = residual; K order i*32 + j, zero padded.
__global__ void cin_split_filter_kernel(const float* __restrict__ w, float* __restrict__ wt, int m, int hk, int H, int NP) {
  const int KP = hk * KB;
  const size_t total = (size_t)NP * KP;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / KP), kk = (int)(idx % KP);
    const int i = kk / KB, j = kk % KB;
    float v = 0.f;
    if (n < H && j < m) v = __ldg(w + ((size_t)i * m + j) * H + n);
    store_split(wt, total, idx, v);
  }
}

// The K loop is cut into accumulation chains of `chunk` K-blocks (tc_ptx.cuh, chain_drain).
//
// Persistent CTAs walk 128-row tiles (two warpgroups x 64 rows); both warpgroups consume every filter stage, a stage is
// released when all eight consumer warps have passed the wgmma.wait that covers it.  While one warpgroup waits for its
// K-block, the other issues its own, and the TMA warp keeps SB stages in flight.
template <int PASSES, int SB, int N>
__global__ void __launch_bounds__(NTHREADS, 1)
cin_fwd_tc_kernel(const __grid_constant__ CUtensorMap tmap_w, const float* __restrict__ x0,
                  const float* __restrict__ xk, float* __restrict__ out, float* __restrict__ pooled, int B, int m,
                  int hk, int logD, int H, int chunk) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int b_tile_bytes = N * 128;
  constexpr int stage_bytes = (PASSES == 3 ? 2 : 1) * b_tile_bytes;
  float* epi = reinterpret_cast<float*>(smem + SB * stage_bytes);
  const uint32_t sbase = smem_u32(smem);
  Ring ring(sbase + SB * stage_bytes + NWG * N * EPI_LD * 4, SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int D = 1 << logD;
  const long long rows_total = (long long)B * D;
  const int n_tiles = (int)((rows_total + TILE_M - 1) / TILE_M);

  ring.init();
  // ============================ TMA producer for the filter tiles ============================
  if (producer_role(warp, lane, [&] {
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
          for (int i = 0; i < hk; ++i) {
            const Ring::Slot slot = ring.acquire(stage_bytes);
            const uint32_t dst = sbase + slot.stage * stage_bytes;
            tma_load_2d(dst, &tmap_w, i * KB, 0, slot.full);
            if (PASSES == 3) tma_load_2d(dst + b_tile_bytes, &tmap_w, i * KB, N, slot.full);
          }
        }
      }))
    return;

  // ============================ consumer warpgroups: A fragments, wgmma, epilogue ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3;
  float* es = epi + wg * N * EPI_LD;
  float dacc[N / 2];
#pragma unroll
  for (int q = 0; q < N / 2; ++q) dacc[q] = 0.f;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long base = (long long)tile * TILE_M + wg * WG_M;
    bool valid[2];
    const float* xkp[2];
    float x0v[2][8];                                   // x0[b, j, d] of this thread's fragment columns j = 8c + t + 4h
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const long long r = base + w * 16 + g + 8 * rr;
      valid[rr] = r < rows_total;
      const int b = valid[rr] ? (int)(r >> logD) : 0;
      const int d = (int)(r & (D - 1));
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int j = 8 * (q >> 1) + t + 4 * (q & 1);
        x0v[rr][q] = (valid[rr] && j < m) ? __ldg(x0 + ((size_t)b * m + j) * D + d) : 0.f;
      }
      xkp[rr] = xk + (size_t)b * hk * D + d;
    }
    float acc[N / 2];
#pragma unroll
    for (int q = 0; q < N / 2; ++q) acc[q] = 0.f;
    for (int i0 = 0; i0 < hk; i0 += chunk) {
      const int i1 = min(hk, i0 + chunk);
      for (int i = i0; i < i1; ++i) {
        const float xi0 = valid[0] ? __ldg(xkp[0] + (size_t)i * D) : 0.f;
        const float xi1 = valid[1] ? __ldg(xkp[1] + (size_t)i * D) : 0.f;
        uint32_t ah[KB / 8][4], al[KB / 8][4];         // A fragments (hi, lo) of the four k-steps of this K-block
#pragma unroll
        for (int c = 0; c < KB / 8; ++c) {
          const float a[4] = {xi0 * x0v[0][2 * c], xi1 * x0v[1][2 * c], xi0 * x0v[0][2 * c + 1], xi1 * x0v[1][2 * c + 1]};
          tf32_split(a, ah[c], al[c]);
        }
        const int s = ring.wait();
        const uint64_t bhi = gmma_desc_kmajor(sbase + s * stage_bytes, 128);
        const uint64_t blo = gmma_desc_kmajor(sbase + s * stage_bytes + b_tile_bytes, 128);
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < KB / 8; ++c) {
          const int sc = (i > i0 || c > 0) ? 1 : 0;
          if (PASSES == 3) mma_3xtf32<N>(dacc, ah[c], al[c], bhi, blo, 2 * c, sc);
          else wgmma_tf32_rs<N>(dacc, ah[c], bhi + 2 * c, sc);
        }
        wgmma_commit();
        wgmma_wait_keep(ah, al);
        ring.release(lane);                            // this warp is done with the stage
      }
      chain_drain(acc, dacc);
    }
    // ---------------- epilogue: fragment -> es[n][row] -> out (B,H,D) and pooled (B,H) ----------------
#pragma unroll
    for (int c = 0; c < N / 8; ++c) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        es[(8 * c + 2 * t + e) * EPI_LD + w * 16 + g] = acc[4 * c + e];
        es[(8 * c + 2 * t + e) * EPI_LD + w * 16 + g + 8] = acc[4 * c + 2 + e];
      }
    }
    wg_bar_sync(1 + wg);
    const int tw = threadIdx.x & 127;
    for (int idx = tw; idx < H * WG_M; idx += 128) {
      const int n = idx / WG_M, row = idx % WG_M;
      const long long r = base + row;
      if (r < rows_total) out[((size_t)(r >> logD) * H + n) * D + (int)(r & (D - 1))] = es[n * EPI_LD + row];
    }
    if (pooled != nullptr) {
      const int nb = WG_M >> logD;                     // samples in this warpgroup's rows (D <= 32 divides 64)
      for (int idx = tw; idx < H * nb; idx += 128) {
        const int n = idx / nb, bl = idx % nb;
        const long long b = (base >> logD) + bl;
        if (b < B) {
          float sum = 0.f;
          for (int d = 0; d < D; ++d) sum += es[n * EPI_LD + bl * D + d];
          pooled[(size_t)b * H + n] = sum;
        }
      }
    }
    wg_bar_sync(1 + wg);
  }
}

// ---- CUDA-core forward for shapes outside the tensor path.  One CTA per sample.
__global__ void __launch_bounds__(256)
cin_fwd_simple_kernel(const float* __restrict__ x0, const float* __restrict__ xk, const float* __restrict__ w,
                      float* __restrict__ out, float* __restrict__ pooled, int B, int m, int hk, int D, int H) {
  extern __shared__ __align__(16) float sm[];
  float* x0s = sm;
  float* xks = sm + m * D;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    for (int i = threadIdx.x; i < m * D; i += blockDim.x) x0s[i] = __ldg(x0 + (size_t)b * m * D + i);
    for (int i = threadIdx.x; i < hk * D; i += blockDim.x) xks[i] = __ldg(xk + (size_t)b * hk * D + i);
    __syncthreads();
    for (int idx = threadIdx.x; idx < H * D; idx += blockDim.x) {
      const int n = idx / D, d = idx % D;
      float acc = 0.f;
      for (int i = 0; i < hk; ++i) {
        const float a = xks[i * D + d];
        const float* wr = w + (size_t)i * m * H + n;
        for (int j = 0; j < m; ++j) acc += (a * x0s[j * D + d]) * __ldg(wr + (size_t)j * H);
      }
      out[(size_t)b * H * D + idx] = acc;
    }
    if (pooled != nullptr) {
      __syncthreads();
      for (int n = threadIdx.x; n < H; n += blockDim.x) {
        float s = 0.f;
        for (int d = 0; d < D; ++d) s += out[((size_t)b * H + n) * D + d];
        pooled[(size_t)b * H + n] = s;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host
static bool tensor_path_ok(int64_t m, int64_t hk, int64_t D, int64_t H) {
  return m >= 1 && m <= KB && hk >= 1 && H >= 1 && H <= 128 && D >= 1 && D <= 32 && (D & (D - 1)) == 0;
}

}  // namespace cin
}  // namespace ctr

using namespace ctr;
using namespace ctr::cin;

extern "C" int64_t ctr_cin_fwd_workspace_bytes(int64_t B, int64_t m, int64_t hk, int64_t D, int64_t H) {
  (void)B;
  if (!tensor_path_ok(m, hk, D, H)) return 0;
  return 2 * (int64_t)pad3(H) * hk * KB * (int64_t)sizeof(float);
}

extern "C" int ctr_cin_fwd(const float* x0, const float* xk, const float* filter, int64_t B, int64_t m, int64_t hk,
                           int64_t D, int64_t H, float* out, float* pooled, int precision, void* workspace,
                           int64_t workspace_bytes, void* stream) {
  CTR_REQUIRE(B >= 0 && m >= 1 && hk >= 1 && D >= 1 && H >= 1, "ctr_cin_fwd: bad sizes B=%lld m=%lld hk=%lld D=%lld H=%lld",
              (long long)B, (long long)m, (long long)hk, (long long)D, (long long)H);
  CTR_UNSUPPORTED(B * D > 0x7fffffffLL || hk * m > (1 << 24), "ctr_cin_fwd: problem too large");
  CTR_REQUIRE(x0 && xk && filter && out, "ctr_cin_fwd: null argument");
  CTR_REQUIRE(precision == 0 || precision == 1, "ctr_cin_fwd: precision must be 0 (3xTF32) or 1 (TF32)");
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  if (!tensor_path_ok(m, hk, D, H)) {
    const size_t smem = sizeof(float) * (size_t)(m + hk) * D;
    CTR_UNSUPPORTED(smem > 200 * 1024, "ctr_cin_fwd: (m+hk)*D too large for the CUDA-core path");
    const int grid = capped_grid(B, (int64_t)sm_count() * 4);
    return launch("ctr_cin_fwd(simple)", cin_fwd_simple_kernel, grid, 256, smem, st, x0, xk, filter, out, pooled, (int)B,
                  (int)m, (int)hk, (int)D, (int)H);
  }
  const int NP = pad3(H);
  int rc = check_workspace("ctr_cin_fwd", "ctr_cin_fwd_workspace_bytes", workspace, workspace_bytes,
                           ctr_cin_fwd_workspace_bytes(B, m, hk, D, H));
  if (rc) return rc;
  float* wt = static_cast<float*>(workspace);
  const int KP = (int)hk * KB;
  rc = launch("ctr_cin_fwd(split filter)", cin_split_filter_kernel, capped_grid(((size_t)NP * KP + 255) / 256, 4096), 256, 0, st, filter,
              wt, (int)m, (int)hk, (int)H, NP);
  if (rc) return rc;
  CUtensorMap tmap;
  rc = encode_2d("ctr_cin_fwd", &tmap, wt, KP, 2 * NP, KB, NP, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  int logD = 0;
  while ((1 << logD) < D) ++logD;
  const long long rows_total = (long long)B * D;
  const int n_tiles = (int)((rows_total + TILE_M - 1) / TILE_M);
  const int grid = capped_grid(n_tiles, sm_count());
  // 3xTF32: 4 stages, chains of 8 K-blocks = 96 chained MMAs before the registers take the sum.  TF32: 6 stages, 32 blocks.
  return with_const<0, 1>(precision, [&](auto P1) {
    constexpr int PASSES = P1 ? 1 : 3, SB = P1 ? 6 : 4, CHUNK = P1 ? 32 : 8;
    return with_const<32, 64, 128>(NP, [&](auto N) {
      return launch("ctr_cin_fwd(wgmma)", cin_fwd_tc_kernel<PASSES, SB, N>, grid, NTHREADS,
                    fwd_smem_bytes(N, PASSES, SB) + 1024, st, tmap, x0, xk, out, pooled, (int)B, (int)m, (int)hk, logD,
                    (int)H, CHUNK);
    });
  });
}

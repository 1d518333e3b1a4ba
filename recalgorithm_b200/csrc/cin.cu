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

constexpr int KB = 32;                    // tf32 per K-block (128 B == swizzle span)
constexpr int NWG = 2;                    // consumer warpgroups per CTA, 64 rows each
constexpr int TILE_M = NWG * WG_M;        // rows per CTA tile
constexpr int NTHREADS = (NWG + 1) * 128;  // + one producer warpgroup (one TMA thread)
constexpr int EPI_LD = WG_M + 4;          // row stride (floats) of the epilogue staging: conflict-free fragment stores

__host__ __device__ inline int fwd_smem_bytes(int N, int passes, int stages) {
  return stages * (passes == 3 ? 2 : 1) * N * 128 + NWG * N * EPI_LD * 4 + 8 * 2 * stages;
}
// wgmma N of the tensor path: hk_1 padded to 32, 64 or 128 (also the row count of the split filter)
static inline int npad(int64_t H) { return H <= 32 ? 32 : H <= 64 ? 64 : 128; }

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
    const float hi = tf32_rna(v);
    wt[idx] = hi;
    wt[total + idx] = v - hi;
  }
}

// Accumulation note: the tensor core adds each K=8 product group into the fp32 accumulator with truncation, so a long
// accumulation chain drifts by ~0.5 ulp per MMA.  The K loop is therefore cut into chunks of `chunk` K-blocks: each chunk
// accumulates from zero and is then added into a second set of fp32 registers (round-to-nearest).
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
  // SWIZZLE_128B operands need 1024-byte aligned tiles: align explicitly (the launch adds 1 KB of slack)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr int b_tile_bytes = N * 128;
  constexpr int stage_bytes = (PASSES == 3 ? 2 : 1) * b_tile_bytes;
  float* epi = reinterpret_cast<float*>(smem + SB * stage_bytes);
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar0 = sbase + SB * stage_bytes + NWG * N * EPI_LD * 4;
  auto full_b = [&](int s) { return bar0 + 8 * s; };
  auto empty_b = [&](int s) { return bar0 + 8 * (SB + s); };

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int D = 1 << logD;
  const long long rows_total = (long long)B * D;
  const int n_tiles = (int)((rows_total + TILE_M - 1) / TILE_M);

  if (threadIdx.x == 0) {
    for (int s = 0; s < SB; ++s) { mbar_init(full_b(s), 1); mbar_init(empty_b(s), NWG * 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= NWG * 4) {
    // ============================ TMA producer for the filter tiles ============================
    setmaxnreg_dec<40>();
    if (warp == NWG * 4 && lane == 0) {
      int s = 0, ph = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        for (int i = 0; i < hk; ++i) {
          mbar_wait(empty_b(s), ph ^ 1);
          const uint32_t dst = sbase + s * stage_bytes;
          mbar_expect_tx(full_b(s), (uint32_t)stage_bytes);
          tma_load_2d(dst, &tmap_w, i * KB, 0, full_b(s));
          if (PASSES == 3) tma_load_2d(dst + b_tile_bytes, &tmap_w, i * KB, N, full_b(s));
          if (++s == SB) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // ============================ consumer warpgroups: A fragments, wgmma, epilogue ============================
  setmaxnreg_inc<232>();
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3;
  float* es = epi + wg * N * EPI_LD;
  int s = 0, ph = 0;
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
        mbar_wait(full_b(s), ph);
        const uint64_t bhi = gmma_desc_kmajor(sbase + s * stage_bytes, 128);
        const uint64_t blo = gmma_desc_kmajor(sbase + s * stage_bytes + b_tile_bytes, 128);
        wgmma_fence();
#pragma unroll
        for (int c = 0; c < KB / 8; ++c) {
          const int sc = (i > i0 || c > 0) ? 1 : 0;
          if (PASSES == 3) {
            // small terms first, the dominant hi*hi term last
            wgmma_tf32_rs<N>(dacc, al[c], bhi + 2 * c, sc);
            wgmma_tf32_rs<N>(dacc, ah[c], blo + 2 * c, 1);
            wgmma_tf32_rs<N>(dacc, ah[c], bhi + 2 * c, 1);
          } else {
            wgmma_tf32_rs<N>(dacc, ah[c], bhi + 2 * c, sc);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int c = 0; c < KB / 8; ++c) { wgmma_keep(ah[c]); wgmma_keep(al[c]); }
        if (lane == 0) mbar_arrive(empty_b(s));        // this warp is done with the stage
        if (++s == SB) { s = 0; ph ^= 1; }
      }
#pragma unroll
      for (int q = 0; q < N / 2; ++q) acc[q] += dacc[q];
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

// ---- CUDA-core backward, data gradients.  One CTA per sample.
//   dz[p,d] = sum_n g[n,d]*W[p,n];  dxk[i,d] += dz*x0[j,d];  dx0[j,d] += dz*xk[i,d]      (p = i*m + j)
__global__ void __launch_bounds__(256)
cin_bwd_dx_kernel(const float* __restrict__ x0, const float* __restrict__ xk, const float* __restrict__ w,
                  const float* __restrict__ g, int B, int m, int hk, int D, int H, float* __restrict__ dx0,
                  float* __restrict__ dxk) {
  extern __shared__ __align__(16) float sm[];
  float* x0s = sm;
  float* xks = x0s + m * D;
  float* gs = xks + hk * D;
  float* dx0s = gs + H * D;
  float* dxks = dx0s + m * D;
  const int d = threadIdx.x % D, pl = threadIdx.x / D, pstep = blockDim.x / D;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    for (int i = threadIdx.x; i < m * D; i += blockDim.x) { x0s[i] = __ldg(x0 + (size_t)b * m * D + i); dx0s[i] = 0.f; }
    for (int i = threadIdx.x; i < hk * D; i += blockDim.x) { xks[i] = __ldg(xk + (size_t)b * hk * D + i); dxks[i] = 0.f; }
    for (int i = threadIdx.x; i < H * D; i += blockDim.x) gs[i] = __ldg(g + (size_t)b * H * D + i);
    __syncthreads();
    if (pl < pstep) {
      for (int p = pl; p < hk * m; p += pstep) {
        const float* wr = w + (size_t)p * H;
        float dz = 0.f;
        for (int n = 0; n < H; ++n) dz += gs[n * D + d] * __ldg(wr + n);
        const int i = p / m, j = p % m;
        atomicAdd(dxks + i * D + d, dz * x0s[j * D + d]);
        atomicAdd(dx0s + j * D + d, dz * xks[i * D + d]);
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < m * D; i += blockDim.x) dx0[(size_t)b * m * D + i] = dx0s[i];
    for (int i = threadIdx.x; i < hk * D; i += blockDim.x) dxk[(size_t)b * hk * D + i] = dxks[i];
  }
}

// ---- CUDA-core backward, filter gradient: dW[p,n] = sum_{b,d} xk[b,i,d]*x0[b,j,d]*g[b,n,d].
// grid (ceil(hk*m / PC), nsplit); block = threads over n; each CTA streams its share of the batch.
constexpr int CIN_PC = 16;
__global__ void __launch_bounds__(256)
cin_bwd_dw_kernel(const float* __restrict__ x0, const float* __restrict__ xk, const float* __restrict__ g, int B, int m,
                  int hk, int D, int H, float* __restrict__ dw) {
  extern __shared__ __align__(16) float sm[];
  float* gs = sm;                         // (H, D+1) padded against bank conflicts
  float* zs = gs + H * (D + 1);           // (PC, D)
  const int p0 = blockIdx.x * CIN_PC;
  const int K = hk * m;
  float acc[CIN_PC];
#pragma unroll
  for (int q = 0; q < CIN_PC; ++q) acc[q] = 0.f;
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    __syncthreads();
    for (int i = threadIdx.x; i < H * D; i += blockDim.x) gs[(i / D) * (D + 1) + i % D] = __ldg(g + (size_t)b * H * D + i);
    for (int i = threadIdx.x; i < CIN_PC * D; i += blockDim.x) {
      const int q = i / D, d = i % D, p = p0 + q;
      float z = 0.f;
      if (p < K) z = __ldg(xk + ((size_t)b * hk + p / m) * D + d) * __ldg(x0 + ((size_t)b * m + p % m) * D + d);
      zs[i] = z;
    }
    __syncthreads();
    for (int n = threadIdx.x; n < H; n += blockDim.x) {     // H <= blockDim in practice: one n per thread
      for (int d = 0; d < D; ++d) {
        const float gv = gs[n * (D + 1) + d];
#pragma unroll
        for (int q = 0; q < CIN_PC; ++q) acc[q] += zs[q * D + d] * gv;
      }
    }
  }
  const int n = threadIdx.x;
  if (n < H) {
#pragma unroll
    for (int q = 0; q < CIN_PC; ++q)
      if (p0 + q < K) atomicAdd(dw + (size_t)(p0 + q) * H + n, acc[q]);
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
  return 2 * (int64_t)npad(H) * hk * KB * (int64_t)sizeof(float);
}

static int check_cin(const char* fn, int64_t B, int64_t m, int64_t hk, int64_t D, int64_t H) {
  CTR_REQUIRE(B >= 0 && m >= 1 && hk >= 1 && D >= 1 && H >= 1, "%s: bad sizes B=%lld m=%lld hk=%lld D=%lld H=%lld", fn,
              (long long)B, (long long)m, (long long)hk, (long long)D, (long long)H);
  CTR_UNSUPPORTED(B * D > 0x7fffffffLL || hk * m > (1 << 24), "%s: problem too large", fn);
  return CTR_OK;
}

extern "C" int ctr_cin_fwd(const float* x0, const float* xk, const float* filter, int64_t B, int64_t m, int64_t hk,
                           int64_t D, int64_t H, float* out, float* pooled, int precision, void* workspace,
                           int64_t workspace_bytes, void* stream) {
  int rc = check_cin("ctr_cin_fwd", B, m, hk, D, H);
  if (rc) return rc;
  CTR_REQUIRE(x0 && xk && filter && out, "ctr_cin_fwd: null argument");
  CTR_REQUIRE(precision == 0 || precision == 1, "ctr_cin_fwd: precision must be 0 (3xTF32) or 1 (TF32)");
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  if (!tensor_path_ok(m, hk, D, H)) {
    const size_t smem = sizeof(float) * (size_t)(m + hk) * D;
    CTR_UNSUPPORTED(smem > 200 * 1024, "ctr_cin_fwd: (m+hk)*D too large for the CUDA-core path");
    if (smem > 48 * 1024)
      CTR_CUDA(cudaFuncSetAttribute(cin_fwd_simple_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = (int)(B < (int64_t)sm_count() * 4 ? B : (int64_t)sm_count() * 4);
    cin_fwd_simple_kernel<<<grid, 256, smem, st>>>(x0, xk, filter, out, pooled, (int)B, (int)m, (int)hk, (int)D, (int)H);
    CTR_CHECK_LAUNCH("ctr_cin_fwd(simple)");
    return CTR_OK;
  }
  const int NP = npad(H);
  const int64_t need = ctr_cin_fwd_workspace_bytes(B, m, hk, D, H);
  CTR_REQUIRE(workspace != nullptr && workspace_bytes >= need,
              "ctr_cin_fwd: workspace of %lld bytes required (ctr_cin_fwd_workspace_bytes), got %lld", (long long)need,
              (long long)workspace_bytes);
  CTR_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 127) == 0, "ctr_cin_fwd: workspace must be 128-byte aligned");
  float* wt = static_cast<float*>(workspace);
  const int KP = (int)hk * KB;
  {
    const long long total = (long long)NP * KP;
    const int grid = (int)((total + 255) / 256 < 4096 ? (total + 255) / 256 : 4096);
    cin_split_filter_kernel<<<grid, 256, 0, st>>>(filter, wt, (int)m, (int)hk, (int)H, NP);
    CTR_CHECK_LAUNCH("ctr_cin_fwd(split filter)");
  }
  EncodeTiledFn enc = encode_tiled();
  if (enc == nullptr) {
    set_error("ctr_cin_fwd: cuTensorMapEncodeTiled is not available from the driver");
    return CTR_ERR_CUDA;
  }
  CUtensorMap tmap;
  const cuuint64_t gdim[2] = {(cuuint64_t)KP, (cuuint64_t)(2 * NP)};
  const cuuint64_t gstride[1] = {(cuuint64_t)KP * sizeof(float)};
  const cuuint32_t box[2] = {(cuuint32_t)KB, (cuuint32_t)NP};
  const cuuint32_t estr[2] = {1, 1};
  CUresult cr = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, wt, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    set_error("ctr_cin_fwd: cuTensorMapEncodeTiled failed with CUresult %d", (int)cr);
    return CTR_ERR_CUDA;
  }
  int logD = 0;
  while ((1 << logD) < D) ++logD;
  const long long rows_total = (long long)B * D;
  const int n_tiles = (int)((rows_total + TILE_M - 1) / TILE_M);
  const int grid = n_tiles < sm_count() ? n_tiles : sm_count();
  // K-blocks per accumulation chain of the 3xTF32 path: 8 blocks = 96 chained MMAs before the registers take the sum
  constexpr int CHUNK3 = 8;
#define CIN_LAUNCH(PASSES_, SB_, N_, CHUNK_)                                                                          \
  {                                                                                                                   \
    const int smem = fwd_smem_bytes(N_, PASSES_, SB_) + 1024;                                                         \
    auto k = cin_fwd_tc_kernel<PASSES_, SB_, N_>;                                                                     \
    CTR_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));                             \
    k<<<grid, NTHREADS, smem, st>>>(tmap, x0, xk, out, pooled, (int)B, (int)m, (int)hk, logD, (int)H, CHUNK_);        \
  }
  if (precision == 0) {
    if (NP == 32) CIN_LAUNCH(3, 4, 32, CHUNK3) else if (NP == 64) CIN_LAUNCH(3, 4, 64, CHUNK3) else CIN_LAUNCH(3, 4, 128, CHUNK3)
  } else {
    if (NP == 32) CIN_LAUNCH(1, 6, 32, 32) else if (NP == 64) CIN_LAUNCH(1, 6, 64, 32) else CIN_LAUNCH(1, 6, 128, 32)
  }
#undef CIN_LAUNCH
  CTR_CHECK_LAUNCH("ctr_cin_fwd(wgmma)");
  return CTR_OK;
}

extern "C" int ctr_cin_bwd_tc_supported(int64_t m, int64_t hk, int64_t D, int64_t H);                 // cin_bwd.cu
int ctr_cin_bwd_tc(const float* x0, const float* xk, const float* filter, const float* g_out, int64_t B, int64_t m,
                   int64_t hk, int64_t D, int64_t H, float* dx0, float* dxk, float* dfilter, void* workspace,
                   cudaStream_t st);                                                                          // cin_bwd.cu

extern "C" int ctr_cin_bwd(const float* x0, const float* xk, const float* filter, const float* g_out, int64_t B,
                           int64_t m, int64_t hk, int64_t D, int64_t H, float* dx0, float* dxk, float* dfilter,
                           void* workspace, int64_t workspace_bytes, void* stream) {
  int rc = check_cin("ctr_cin_bwd", B, m, hk, D, H);
  if (rc) return rc;
  CTR_REQUIRE(x0 && xk && filter && g_out && dx0 && dxk && dfilter, "ctr_cin_bwd: null argument");
  CTR_UNSUPPORTED(D > 256 || H > 256, "ctr_cin_bwd: D=%lld H=%lld too large", (long long)D, (long long)H);
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(dfilter, 0, sizeof(float) * hk * m * H, st));
  if (B == 0) return CTR_OK;
  if (ctr_cin_bwd_tc_supported(m, hk, D, H)) {
    const int64_t need = ctr_cin_bwd_workspace_bytes(B, m, hk, D, H);
    CTR_REQUIRE(workspace != nullptr && workspace_bytes >= need,
                "ctr_cin_bwd: workspace of %lld bytes required (ctr_cin_bwd_workspace_bytes), got %lld", (long long)need,
                (long long)workspace_bytes);
    CTR_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 127) == 0, "ctr_cin_bwd: workspace must be 128-byte aligned");
    return ctr_cin_bwd_tc(x0, xk, filter, g_out, B, m, hk, D, H, dx0, dxk, dfilter, workspace, st);
  }
  {
    const size_t smem = sizeof(float) * (size_t)(2 * (m + hk) + H) * D;
    CTR_UNSUPPORTED(smem > 200 * 1024, "ctr_cin_bwd: shared memory need %zu B too large", smem);
    if (smem > 48 * 1024)
      CTR_CUDA(cudaFuncSetAttribute(cin_bwd_dx_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int grid = (int)(B < (int64_t)sm_count() * 4 ? B : (int64_t)sm_count() * 4);
    cin_bwd_dx_kernel<<<grid, 256, smem, st>>>(x0, xk, filter, g_out, (int)B, (int)m, (int)hk, (int)D, (int)H, dx0, dxk);
    CTR_CHECK_LAUNCH("ctr_cin_bwd(dx)");
  }
  {
    const size_t smem = sizeof(float) * (size_t)(H * (D + 1) + CIN_PC * D);
    CTR_UNSUPPORTED(smem > 200 * 1024, "ctr_cin_bwd: shared memory need %zu B too large", smem);
    if (smem > 48 * 1024)
      CTR_CUDA(cudaFuncSetAttribute(cin_bwd_dw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int gx = (int)((hk * m + CIN_PC - 1) / CIN_PC);
    int gy = (int)((int64_t)sm_count() * 4 / gx);
    if (gy < 1) gy = 1;
    if (gy > B) gy = (int)B;
    cin_bwd_dw_kernel<<<dim3(gx, gy), 256, smem, st>>>(x0, xk, g_out, (int)B, (int)m, (int)hk, (int)D, (int)H, dfilter);
    CTR_CHECK_LAUNCH("ctr_cin_bwd(dw)");
  }
  return CTR_OK;
}

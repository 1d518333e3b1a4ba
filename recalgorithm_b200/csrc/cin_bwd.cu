// Row CIN, backward on the tensor cores (wgmma) -- gradients of xDeepFM/cin_layer.py:17-30.
//
//   out[b,n,d] = sum_{i,j} xk[b,i,d] x0[b,j,d] W[(i,j),n]            g = dL/dout  (B,H,D)
//   dZ[r,(i,j)] = sum_n g[b,n,d] W[(i,j),n]      (r = (b,d))
//   dxk[b,i,d]  = sum_j dZ[r,(i,j)] x0[b,j,d]        dx0[b,j,d] = sum_i dZ[r,(i,j)] xk[b,i,d]
//   dW[(i,j),n] = sum_r xk[b,i,d] x0[b,j,d] g[b,n,d]
//
// Two kernels.  In both the operand the threads generate is the wgmma A operand, held in registers in the A-fragment
// layout, and the streamed operand is delivered by TMA into swizzled shared memory through an mbarrier pipeline;
// 3xTF32 split for fp32-class accuracy (see cin.cu and tc_ptx.cuh for the accuracy notes):
//
//  dX kernel   GEMM dZ_i[64 rows x 64 (i,j)] = G[64 x H] . W^T[H x 64]   for two i per step
//     A = G: each thread loads the g values of its two rows once per tile into registers;
//     B = W rows (i0*m .. i0*m+63) x H, K-major in the filter's native layout, TMA-streamed (4-D box = HP/32 swizzled sub-tiles);
//     dZ stays in the accumulator registers: the thread does both contractions on its fragment (dxk: dot with its x0
//     registers + a reduction over the 4 threads that share a row; dx0: axpy into register accumulators).
//
//  dW kernel   GEMM dW_blk[64 (i,j) x H] += Z^T[64 (i,j) x D] . G_b^T[D x H]   for every sample b
//     A = Z^T: thread (i,j) forms xk[b,i,d] * x0[b,j,d] for the d of its fragment columns;
//     B = g[b] as [H rows x D] K-major tiles (TMA 3-D box, swizzle width = D*4 bytes);
//     each CTA owns 4 consecutive i (two warpgroups x 64 (i,j) rows) and a slice of the batch; accumulation chains are cut
//     every `chunk` samples and added into fp32 registers (round-to-nearest); one atomic add per element at the end.
//
// Shapes outside the tensor path's limits (m > 32, hk_1 > 128, D not 8, 16 or 32) run the CUDA-core kernels below.
#include <stdlib.h>

#include "tc_ptx.cuh"

namespace ctr {
namespace cinb {
using namespace ctr::tc;

// ================================================================================================= prep kernels
// filter (hk*m, H) -> ws[2][KRP][HP]  (tf32-rounded value | residual), zero padded rows/cols.
__global__ void split_filter_native_kernel(const float* __restrict__ w, float* __restrict__ ws, int K, int H, int KRP, int HP) {
  const size_t total = (size_t)KRP * HP;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int row = (int)(idx / HP), n = (int)(idx % HP);
    float v = 0.f;
    if (row < K && n < H) v = __ldg(w + (size_t)row * H + n);
    store_split(ws, total, idx, v);
  }
}
// g (B,H,D) -> gs[2][B][H][D]
__global__ void split_grad_kernel(const float* __restrict__ g, float* __restrict__ gs, size_t total) {
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x)
    store_split(gs, total, idx, __ldg(g + idx));
}

// ================================================================================================= dX kernel
constexpr int DX_IPS = 2;           // i's per step
constexpr int DX_N = DX_IPS * KB;   // 64 columns of dZ per step (wgmma N)
constexpr int DX_TILE = NWG * WG_M; // rows per CTA tile

template <int SB, int NKB>
__global__ void __launch_bounds__(NTHREADS, 1)
cin_bwd_dx_tc_kernel(const __grid_constant__ CUtensorMap tmap_w, const float* __restrict__ x0,
                     const float* __restrict__ xk, const float* __restrict__ g, float* __restrict__ dx0,
                     float* __restrict__ dxk, int B, int m, int hk, int logD, int H, int KRP) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int HP = NKB * KB;
  constexpr int b_copy_bytes = NKB * DX_N * 128;           // one (hi or lo) copy: NKB sub-tiles of [64 rows x 128 B]
  constexpr int stage_bytes = 2 * b_copy_bytes;
  const uint32_t sbase = smem_u32(smem);
  Ring ring(sbase + SB * stage_bytes, SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int D = 1 << logD;
  const long long rows_total = (long long)B * D;
  const int num_tiles = (int)((rows_total + DX_TILE - 1) / DX_TILE);
  const int nsteps = (hk + DX_IPS - 1) / DX_IPS;

  ring.init();
  // ============================ TMA: filter rows of i0 and i0+1 (hi and lo copies) ============================
  if (producer_role(warp, lane, [&] {
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
          for (int st = 0; st < nsteps; ++st) {
            const Ring::Slot slot = ring.acquire(stage_bytes);
            const uint32_t dst = sbase + slot.stage * stage_bytes;
            tma_load_4d(dst, &tmap_w, 0, st * DX_IPS * m, 0, 0, slot.full);
            tma_load_4d(dst + b_copy_bytes, &tmap_w, 0, KRP + st * DX_IPS * m, 0, 0, slot.full);
          }
        }
      }))
    return;

  // ============================ consumers: G fragments once per tile, then dZ of two i per step ============================
  const int wg = warp >> 2, w = warp & 3, gq = lane >> 2, t = lane & 3;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const long long base = (long long)tile * DX_TILE + wg * WG_M;
    bool valid[2];
    int bb[2], dd[2];
    float x0v[2][8], dx0acc[2][8];                   // fragment columns j = 8c + 2t + e  ->  [2c + e]
    uint32_t gh[HP / 8][4], gl[HP / 8][4];           // A fragments of G (hi, lo): k-step s, columns n = 8s + t (+4)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const long long r = base + w * 16 + gq + 8 * rr;
      valid[rr] = r < rows_total;
      bb[rr] = valid[rr] ? (int)(r >> logD) : 0;
      dd[rr] = (int)(r & (D - 1));
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int j = 8 * (q >> 1) + 2 * t + (q & 1);
        x0v[rr][q] = (valid[rr] && j < m) ? __ldg(x0 + ((size_t)bb[rr] * m + j) * D + dd[rr]) : 0.f;
        dx0acc[rr][q] = 0.f;
      }
    }
#pragma unroll
    for (int ks = 0; ks < HP / 8; ++ks) {
      float ga[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int rr = q & 1, n = 8 * ks + t + 4 * (q >> 1);
        ga[q] = (valid[rr] && n < H) ? __ldg(g + ((size_t)bb[rr] * H + n) * D + dd[rr]) : 0.f;
      }
      tf32_split(ga, gh[ks], gl[ks]);                // split once per tile: the wgmmas in flight read these registers
    }
    auto load_xi = [&](int i0, float (&xi)[2][DX_IPS]) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr)
#pragma unroll
        for (int h = 0; h < DX_IPS; ++h)
          xi[rr][h] = (valid[rr] && i0 + h < hk) ? __ldg(xk + ((size_t)bb[rr] * hk + i0 + h) * D + dd[rr]) : 0.f;
    };
    float xi[2][DX_IPS];
    load_xi(0, xi);
    for (int st = 0; st < nsteps; ++st) {
      const int i0 = st * DX_IPS;
      const int s = ring.wait();
      const uint64_t bhi = gmma_desc_kmajor(sbase + s * stage_bytes, 128);
      const uint64_t blo = gmma_desc_kmajor(sbase + s * stage_bytes + b_copy_bytes, 128);
      float dz[DX_N / 2];
#pragma unroll
      for (int q = 0; q < DX_N / 2; ++q) dz[q] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < HP / 8; ++ks) {
        // sub-tile kb of a copy starts DX_N*128 bytes (>>4 = 512) further
        const uint64_t off = (uint64_t)((ks >> 2) * (DX_N * 128 / 16) + 2 * (ks & 3));
        mma_3xtf32<DX_N>(dz, gh[ks], gl[ks], bhi, blo, off, ks > 0 ? 1 : 0);
      }
      wgmma_commit();
      float xin[2][DX_IPS];                            // the next step's xk values, loaded while this group runs
      load_xi(i0 + DX_IPS, xin);
      wgmma_wait<0>();                                 // gh / gl are not rewritten before the next tile, after this wait
      ring.release(lane);
      // dz[4c + 2rr + e] = dZ[row rr][column 8c + 2t + e]; columns 0..31 belong to i0, 32..63 to i0 + 1
#pragma unroll
      for (int h = 0; h < DX_IPS; ++h) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          float p = 0.f;
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const float v = dz[4 * (4 * h + (q >> 1)) + 2 * rr + (q & 1)];
            p += v * x0v[rr][q];                       // x0v[j >= m] == 0 masks the rows that belong to the next i
            dx0acc[rr][q] += v * xi[rr][h];            // xi == 0 for i >= hk
          }
          p += __shfl_xor_sync(0xffffffffu, p, 1);
          p += __shfl_xor_sync(0xffffffffu, p, 2);
          if (t == 0 && valid[rr] && i0 + h < hk) dxk[((size_t)bb[rr] * hk + i0 + h) * D + dd[rr]] = p;
        }
      }
#pragma unroll
      for (int rr = 0; rr < 2; ++rr)
#pragma unroll
        for (int h = 0; h < DX_IPS; ++h) xi[rr][h] = xin[rr][h];
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int j = 8 * (q >> 1) + 2 * t + (q & 1);
        if (valid[rr] && j < m) dx0[((size_t)bb[rr] * m + j) * D + dd[rr]] = dx0acc[rr][q];
      }
    }
  }
}

// ================================================================================================= dW kernel
constexpr int DW_IPC = NWG * 2;     // i per CTA: each warpgroup owns 64 (i,j) rows = 2 i x 32 j

template <int N, int D>
__global__ void __launch_bounds__(NTHREADS, 1)
cin_bwd_dw_tc_kernel(const __grid_constant__ CUtensorMap tmap_g, const float* __restrict__ x0,
                     const float* __restrict__ xk, float* __restrict__ dw, int B, int m, int hk, int H,
                     int ngroups, int nslices, int chunk, int SB) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int row_bytes = D * 4;                         // one sample's D values of one n-row (= swizzle width)
  constexpr int b_copy_bytes = N * row_bytes;
  constexpr int stage_bytes = 2 * b_copy_bytes;
  const uint32_t sbase = smem_u32(smem);
  Ring ring(sbase + SB * stage_bytes, SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int group = blockIdx.x % ngroups;
  int b_beg, b_end;
  batch_slice(blockIdx.x / ngroups, nslices, B, b_beg, b_end);

  ring.init();
  // ============================ TMA: g[b] as [N rows x D] tiles (hi and lo) ============================
  if (producer_role(warp, lane, [&] {
        for (int b = b_beg; b < b_end; ++b) {
          const Ring::Slot slot = ring.acquire(stage_bytes);
          const uint32_t dst = sbase + slot.stage * stage_bytes;
          tma_load_3d(dst, &tmap_g, 0, 0, b, slot.full);
          tma_load_3d(dst + b_copy_bytes, &tmap_g, 0, 0, B + b, slot.full);
        }
      }))
    return;

  // ============================ (i,j)-row owners: Z^T fragments, wgmma, chunk drains, final reduction ============================
  const int wg = warp >> 2, w = warp & 3, gq = lane >> 2, t = lane & 3;
  const int i = group * DW_IPC + wg * 2 + (w >> 1);        // rows 16w + gq (+8) of the warpgroup = i_local * 32 + j
  const int j0 = (w & 1) * 16 + gq, j1 = j0 + 8;
  const bool live0 = i < hk && j0 < m, live1 = i < hk && j1 < m;   // padding rows produce zeros and are never stored
  float acc[N / 2], dacc[N / 2];
#pragma unroll
  for (int q = 0; q < N / 2; ++q) { acc[q] = 0.f; dacc[q] = 0.f; }
  // A fragments (hi, lo) of the D/8 k-steps of sample b; fragment columns d = 8k + t + 4h  ->  [2k + h]
  auto form = [&](int b, uint32_t (&fh)[D / 8][4], uint32_t (&fl)[D / 8][4]) {
    float xa[D / 4], xb0[D / 4], xb1[D / 4];
#pragma unroll
    for (int q = 0; q < D / 4; ++q) {
      const int d = 8 * (q >> 1) + t + 4 * (q & 1);
      xa[q] = i < hk ? __ldg(xk + ((size_t)b * hk + i) * D + d) : 0.f;
      xb0[q] = live0 ? __ldg(x0 + ((size_t)b * m + j0) * D + d) : 0.f;
      xb1[q] = live1 ? __ldg(x0 + ((size_t)b * m + j1) * D + d) : 0.f;
    }
#pragma unroll
    for (int k = 0; k < D / 8; ++k) {
      const float a[4] = {xa[2 * k] * xb0[2 * k], xa[2 * k] * xb1[2 * k], xa[2 * k + 1] * xb0[2 * k + 1],
                          xa[2 * k + 1] * xb1[2 * k + 1]};
      tf32_split(a, fh[k], fl[k]);
    }
  };
  uint32_t ah[D / 8][4], al[D / 8][4];
  if (b_end > b_beg) form(b_beg, ah, al);
  for (int b = b_beg; b < b_end; ++b) {
    const bool chunk_start = chain_first(b - b_beg, chunk);
    const int s = ring.wait();
    const uint64_t bhi = gmma_desc_kmajor(sbase + s * stage_bytes, row_bytes);
    const uint64_t blo = gmma_desc_kmajor(sbase + s * stage_bytes + b_copy_bytes, row_bytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < D / 8; ++k) mma_3xtf32<N>(dacc, ah[k], al[k], bhi, blo, 2 * k, (chunk_start && k == 0) ? 0 : 1);
    wgmma_commit();
    // the next sample's loads and fragments overlap this group (ah / al stay live until after the wait)
    uint32_t bh[D / 8][4], bl[D / 8][4];
    form(b + 1 < b_end ? b + 1 : b, bh, bl);
    wgmma_wait_keep(ah, al);
    ring.release(lane);
    if (chain_last(b - b_beg, b_end - b_beg, chunk)) chain_drain(acc, dacc);
#pragma unroll
    for (int k = 0; k < D / 8; ++k)
#pragma unroll
      for (int q = 0; q < 4; ++q) { ah[k][q] = bh[k][q]; al[k][q] = bl[k][q]; }
  }
  if (b_end > b_beg) {
#pragma unroll
    for (int c = 0; c < N / 8; ++c) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = 8 * c + 2 * t + e;
        if (n < H) {
          if (live0) atomicAdd(dw + ((size_t)i * m + j0) * H + n, acc[4 * c + e]);
          if (live1) atomicAdd(dw + ((size_t)i * m + j1) * H + n, acc[4 * c + 2 + e]);
        }
      }
    }
  }
}

// ================================================================================================= CUDA-core path
// ---- data gradients.  One CTA per sample.
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

// ---- filter gradient: dW[p,n] = sum_{b,d} xk[b,i,d]*x0[b,j,d]*g[b,n,d].
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

// Shapes the tensor-core backward serves; everything else goes to the CUDA-core kernels.
static bool tensor_path_ok(int64_t m, int64_t hk, int64_t D, int64_t H) {
  return m >= 1 && m <= 32 && hk >= 1 && H >= 1 && H <= 128 && (D == 8 || D == 16 || D == 32);
}

}  // namespace cinb
}  // namespace ctr

using namespace ctr;
using namespace ctr::cinb;

extern "C" int64_t ctr_cin_bwd_workspace_bytes(int64_t B, int64_t m, int64_t hk, int64_t D, int64_t H) {
  if (!tensor_path_ok(m, hk, D, H)) return 0;
  const int64_t HP = pad_to(H, 32), KRP = (hk + 2) * m + 32;
  return ((2 * KRP + m) * HP + 2 * B * H * D) * (int64_t)sizeof(float);
}

extern "C" int ctr_cin_bwd(const float* x0, const float* xk, const float* filter, const float* g_out, int64_t B,
                           int64_t m, int64_t hk, int64_t D, int64_t H, float* dx0, float* dxk, float* dfilter,
                           void* workspace, int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_cin_bwd";
  CTR_REQUIRE(B >= 0 && m >= 1 && hk >= 1 && D >= 1 && H >= 1, "ctr_cin_bwd: bad sizes B=%lld m=%lld hk=%lld D=%lld H=%lld",
              (long long)B, (long long)m, (long long)hk, (long long)D, (long long)H);
  CTR_UNSUPPORTED(B * D > 0x7fffffffLL || hk * m > (1 << 24), "ctr_cin_bwd: problem too large");
  CTR_REQUIRE(x0 && xk && filter && g_out && dx0 && dxk && dfilter, "ctr_cin_bwd: null argument");
  CTR_UNSUPPORTED(D > 256 || H > 256, "ctr_cin_bwd: D=%lld H=%lld too large", (long long)D, (long long)H);
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(dfilter, 0, sizeof(float) * hk * m * H, st));
  if (B == 0) return CTR_OK;
  const int sms = sm_count();
  int rc;
  if (!tensor_path_ok(m, hk, D, H)) {
    const size_t smem_dx = sizeof(float) * (size_t)(2 * (m + hk) + H) * D;
    CTR_UNSUPPORTED(smem_dx > 200 * 1024, "ctr_cin_bwd: shared memory need %zu B too large", smem_dx);
    const int grid = capped_grid(B, (int64_t)sms * 4);
    rc = launch("ctr_cin_bwd(dx)", cin_bwd_dx_kernel, grid, 256, smem_dx, st, x0, xk, filter, g_out, (int)B, (int)m,
                (int)hk, (int)D, (int)H, dx0, dxk);
    if (rc) return rc;
    const size_t smem_dw = sizeof(float) * (size_t)(H * (D + 1) + CIN_PC * D);
    CTR_UNSUPPORTED(smem_dw > 200 * 1024, "ctr_cin_bwd: shared memory need %zu B too large", smem_dw);
    const int gx = (int)((hk * m + CIN_PC - 1) / CIN_PC);
    int gy = (int)((int64_t)sms * 4 / gx);
    if (gy < 1) gy = 1;
    if (gy > B) gy = (int)B;
    return launch("ctr_cin_bwd(dw)", cin_bwd_dw_kernel, dim3(gx, gy), 256, smem_dw, st, x0, xk, g_out, (int)B, (int)m,
                  (int)hk, (int)D, (int)H, dfilter);
  }
  rc = check_workspace(fn, "ctr_cin_bwd_workspace_bytes", workspace, workspace_bytes,
                       ctr_cin_bwd_workspace_bytes(B, m, hk, D, H));
  if (rc) return rc;
  const int HP = (int)pad_to(H, 32), KRP = (int)((hk + 2) * m + 32);
  const int NP = pad3(H);                                   // wgmma N of the dW kernel
  float* ws_w = static_cast<float*>(workspace);
  float* ws_g = ws_w + (size_t)(2 * KRP + m) * HP;          // + m rows so the i-in-step window of the lo copy stays inside
  rc = launch("ctr_cin_bwd(split filter)", split_filter_native_kernel, capped_grid(((size_t)KRP * HP + 255) / 256, 2048), 256, 0, st,
              filter, ws_w, (int)(hk * m), (int)H, KRP, HP);
  if (rc) return rc;
  const size_t tg = (size_t)B * H * D;
  rc = launch("ctr_cin_bwd(split grad)", split_grad_kernel, capped_grid((tg + 255) / 256, 4096), 256, 0, st, g_out, ws_g, tg);
  if (rc) return rc;
  int logD = 0;
  while ((1 << logD) < D) ++logD;
  // ---- dX: filter as a 4-D tensor (n_inner 32 | row | i-in-step (stride m rows) | n_outer) so one box lands as
  //      HP/32 K-major [64 rows x 128 B] swizzled sub-tiles holding the rows of i0 and i0+1
  {
    CUtensorMap tmap;
    const cuuint64_t gdim[4] = {32, (cuuint64_t)(2 * KRP), (cuuint64_t)DX_IPS, (cuuint64_t)(HP / 32)};
    const cuuint64_t gstr[3] = {(cuuint64_t)HP * sizeof(float), (cuuint64_t)m * HP * sizeof(float), 32 * sizeof(float)};
    const cuuint32_t box[4] = {32, 32, (cuuint32_t)DX_IPS, (cuuint32_t)(HP / 32)};
    rc = encode_tmap(fn, &tmap, 4, ws_w, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    constexpr int SB = 3;
    const int nkb = HP / 32;
    const int smem = SB * 2 * nkb * DX_N * 128 + 8 * 2 * SB + 1024;
    const long long rows = (long long)B * D;
    const int tiles = (int)((rows + DX_TILE - 1) / DX_TILE);
    const int grid = capped_grid(tiles, sms);
    rc = with_const<1, 2, 3, 4>(nkb, [&](auto NKB) {
      return launch("ctr_cin_bwd(dx, wgmma)", cin_bwd_dx_tc_kernel<SB, NKB>, grid, NTHREADS, smem, st, tmap, x0, xk, g_out,
                    dx0, dxk, (int)B, (int)m, (int)hk, logD, (int)H, KRP);
    });
    if (rc) return rc;
  }
  // ---- dW: g (hi | lo stacked along the batch axis) as a 3-D tensor (d | n | b); box = one sample's [NP x D] tile
  //      (rows n >= H are out of bounds and arrive as zeros)
  CUtensorMap tmap;
  const cuuint64_t gdim[3] = {(cuuint64_t)D, (cuuint64_t)H, (cuuint64_t)(2 * B)};
  const cuuint64_t gstr[2] = {(cuuint64_t)D * sizeof(float), (cuuint64_t)H * D * sizeof(float)};
  const cuuint32_t box[3] = {(cuuint32_t)D, (cuuint32_t)NP, 1};
  const CUtensorMapSwizzle sw = D == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : D == 16 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                                               : CU_TENSOR_MAP_SWIZZLE_32B;
  rc = encode_tmap(fn, &tmap, 3, ws_g, gdim, gstr, box, sw);
  if (rc) return rc;
  const int stage_bytes = 2 * NP * (int)D * 4;
  int sb = (192 * 1024) / stage_bytes;                        // as many stages as 192 KB of shared memory hold, at most 8
  if (sb > 8) sb = 8;
  const int smem = sb * stage_bytes + 8 * 2 * sb + 1024;
  const int ngroups = (int)((hk + DW_IPC - 1) / DW_IPC);
  const int nslices = batch_slices(sms, ngroups, B);
  const int grid = ngroups * nslices;
  const int chunk = (int)(256 / D);                          // 96 chained MMAs per accumulator before a drain
  return with_const<32, 64, 128>(NP, [&](auto N) {
    return with_const<8, 16, 32>((int)D, [&](auto DD) {
      return launch("ctr_cin_bwd(dw, wgmma)", cin_bwd_dw_tc_kernel<N, DD>, grid, NTHREADS, smem, st, tmap, x0, xk,
                    dfilter, (int)B, (int)m, (int)hk, (int)H, ngroups, nslices, chunk, sb);
    });
  });
}

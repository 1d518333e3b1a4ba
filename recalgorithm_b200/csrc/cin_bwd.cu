// Row CIN, backward on the tensor cores (wgmma) -- gradients of xDeepFM/cin_layer.py:17-30.
//
//   out[b,n,d] = sum_{i,j} xk[b,i,d] x0[b,j,d] W[(i,j),n]            g = dL/dout  (B,H,D)
//   dZ[r,(i,j)] = sum_n g[b,n,d] W[(i,j),n]      (r = (b,d))
//   dxk[b,i,d]  = sum_j dZ[r,(i,j)] x0[b,j,d]        dx0[b,j,d] = sum_i dZ[r,(i,j)] xk[b,i,d]
//   dW[(i,j),n] = sum_r xk[b,i,d] x0[b,j,d] g[b,n,d]
//
// Two kernels.  In both the operand the threads generate is the wgmma A operand, held in registers in the A-fragment
// layout, and the streamed operand is delivered by TMA into swizzled shared memory through an mbarrier pipeline;
// 3xTF32 split for fp32-class accuracy (see cin.cu for the accuracy notes):
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
#include <stdlib.h>

#include "tc_ptx.cuh"

namespace ctr {
namespace cinb {
using namespace ctr::tc;

constexpr int KB = 32;
constexpr int NWG = 2;                      // consumer warpgroups per CTA
constexpr int NTHREADS = (NWG + 1) * 128;   // + one producer warpgroup (one TMA thread)

// ================================================================================================= prep kernels
// filter (hk*m, H) -> ws[2][KRP][HP]  (tf32-rounded value | residual), zero padded rows/cols.
__global__ void split_filter_native_kernel(const float* __restrict__ w, float* __restrict__ ws, int K, int H, int KRP, int HP) {
  const size_t total = (size_t)KRP * HP;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int row = (int)(idx / HP), n = (int)(idx % HP);
    float v = 0.f;
    if (row < K && n < H) v = __ldg(w + (size_t)row * H + n);
    const float hi = tf32_rna(v);
    ws[idx] = hi;
    ws[total + idx] = v - hi;
  }
}
// g (B,H,D) -> gs[2][B][H][D]
__global__ void split_grad_kernel(const float* __restrict__ g, float* __restrict__ gs, size_t total) {
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const float v = __ldg(g + idx);
    const float hi = tf32_rna(v);
    gs[idx] = hi;
    gs[total + idx] = v - hi;
  }
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
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr int HP = NKB * KB;
  constexpr int b_copy_bytes = NKB * DX_N * 128;           // one (hi or lo) copy: NKB sub-tiles of [64 rows x 128 B]
  constexpr int stage_bytes = 2 * b_copy_bytes;
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar0 = sbase + SB * stage_bytes;
  auto full_b = [&](int s) { return bar0 + 8 * s; };
  auto empty_b = [&](int s) { return bar0 + 8 * (SB + s); };

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int D = 1 << logD;
  const long long rows_total = (long long)B * D;
  const int num_tiles = (int)((rows_total + DX_TILE - 1) / DX_TILE);
  const int nsteps = (hk + DX_IPS - 1) / DX_IPS;

  if (threadIdx.x == 0) {
    for (int s = 0; s < SB; ++s) { mbar_init(full_b(s), 1); mbar_init(empty_b(s), NWG * 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= NWG * 4) {
    // ============================ TMA: filter rows of i0 and i0+1 (hi and lo copies) ============================
    setmaxnreg_dec<40>();
    if (warp == NWG * 4 && lane == 0) {
      int s = 0, ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        for (int st = 0; st < nsteps; ++st) {
          mbar_wait(empty_b(s), ph ^ 1);
          const uint32_t dst = sbase + s * stage_bytes;
          mbar_expect_tx(full_b(s), (uint32_t)stage_bytes);
          tma_load_4d(dst, &tmap_w, 0, st * DX_IPS * m, 0, 0, full_b(s));
          tma_load_4d(dst + b_copy_bytes, &tmap_w, 0, KRP + st * DX_IPS * m, 0, 0, full_b(s));
          if (++s == SB) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // ============================ consumers: G fragments once per tile, then dZ of two i per step ============================
  setmaxnreg_inc<232>();
  const int wg = warp >> 2, w = warp & 3, gq = lane >> 2, t = lane & 3;
  int s = 0, ph = 0;
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
      mbar_wait(full_b(s), ph);
      const uint64_t bhi = gmma_desc_kmajor(sbase + s * stage_bytes, 128);
      const uint64_t blo = gmma_desc_kmajor(sbase + s * stage_bytes + b_copy_bytes, 128);
      float dz[DX_N / 2];
#pragma unroll
      for (int q = 0; q < DX_N / 2; ++q) dz[q] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < HP / 8; ++ks) {
        // sub-tile kb of a copy starts DX_N*128 bytes (>>4 = 512) further; small terms first
        const uint64_t off = (uint64_t)((ks >> 2) * (DX_N * 128 / 16) + 2 * (ks & 3));
        wgmma_tf32_rs<DX_N>(dz, gl[ks], bhi + off, ks > 0 ? 1 : 0);
        wgmma_tf32_rs<DX_N>(dz, gh[ks], blo + off, 1);
        wgmma_tf32_rs<DX_N>(dz, gh[ks], bhi + off, 1);
      }
      wgmma_commit();
      float xin[2][DX_IPS];                            // the next step's xk values, loaded while this group runs
      load_xi(i0 + DX_IPS, xin);
      wgmma_wait<0>();                                 // gh / gl are not rewritten before the next tile, after this wait
      if (lane == 0) mbar_arrive(empty_b(s));
      if (++s == SB) { s = 0; ph ^= 1; }
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
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr int row_bytes = D * 4;                         // one sample's D values of one n-row (= swizzle width)
  constexpr int b_copy_bytes = N * row_bytes;
  constexpr int stage_bytes = 2 * b_copy_bytes;
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar0 = sbase + SB * stage_bytes;
  auto full_b = [&](int s) { return bar0 + 8 * s; };
  auto empty_b = [&](int s) { return bar0 + 8 * (SB + s); };

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int group = blockIdx.x % ngroups, slice = blockIdx.x / ngroups;
  const int per_slice = (B + nslices - 1) / nslices;
  const int b_beg = min(B, slice * per_slice), b_end = min(B, b_beg + per_slice);

  if (threadIdx.x == 0) {
    for (int s = 0; s < SB; ++s) { mbar_init(full_b(s), 1); mbar_init(empty_b(s), NWG * 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= NWG * 4) {
    // ============================ TMA: g[b] as [N rows x D] tiles (hi and lo) ============================
    setmaxnreg_dec<40>();
    if (warp == NWG * 4 && lane == 0) {
      int s = 0, ph = 0;
      for (int b = b_beg; b < b_end; ++b) {
        mbar_wait(empty_b(s), ph ^ 1);
        const uint32_t dst = sbase + s * stage_bytes;
        mbar_expect_tx(full_b(s), (uint32_t)stage_bytes);
        tma_load_3d(dst, &tmap_g, 0, 0, b, full_b(s));
        tma_load_3d(dst + b_copy_bytes, &tmap_g, 0, 0, B + b, full_b(s));
        if (++s == SB) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ============================ (i,j)-row owners: Z^T fragments, wgmma, chunk drains, final reduction ============================
  setmaxnreg_inc<232>();
  const int wg = warp >> 2, w = warp & 3, gq = lane >> 2, t = lane & 3;
  const int i = group * DW_IPC + wg * 2 + (w >> 1);        // rows 16w + gq (+8) of the warpgroup = i_local * 32 + j
  const int j0 = (w & 1) * 16 + gq, j1 = j0 + 8;
  const bool live0 = i < hk && j0 < m, live1 = i < hk && j1 < m;   // padding rows produce zeros and are never stored
  float acc[N / 2], dacc[N / 2];
#pragma unroll
  for (int q = 0; q < N / 2; ++q) { acc[q] = 0.f; dacc[q] = 0.f; }
  int s = 0, ph = 0;
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
    const bool chunk_start = (b - b_beg) % chunk == 0;
    mbar_wait(full_b(s), ph);
    const uint64_t bhi = gmma_desc_kmajor(sbase + s * stage_bytes, row_bytes);
    const uint64_t blo = gmma_desc_kmajor(sbase + s * stage_bytes + b_copy_bytes, row_bytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < D / 8; ++k) {
      const int sc = (chunk_start && k == 0) ? 0 : 1;
      wgmma_tf32_rs<N>(dacc, al[k], bhi + 2 * k, sc);
      wgmma_tf32_rs<N>(dacc, ah[k], blo + 2 * k, 1);
      wgmma_tf32_rs<N>(dacc, ah[k], bhi + 2 * k, 1);
    }
    wgmma_commit();
    // the next sample's loads and fragments overlap this group (ah / al stay live until after the wait)
    uint32_t bh[D / 8][4], bl[D / 8][4];
    form(b + 1 < b_end ? b + 1 : b, bh, bl);
    wgmma_wait<0>();
#pragma unroll
    for (int k = 0; k < D / 8; ++k) { wgmma_keep(ah[k]); wgmma_keep(al[k]); }
    if (lane == 0) mbar_arrive(empty_b(s));
    if (++s == SB) { s = 0; ph ^= 1; }
    if ((b + 1 - b_beg) % chunk == 0 || b + 1 == b_end) {
#pragma unroll
      for (int q = 0; q < N / 2; ++q) acc[q] += dacc[q];
    }
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

static int64_t pad_to(int64_t v, int64_t q) { return (v + q - 1) / q * q; }

}  // namespace cinb
}  // namespace ctr

using namespace ctr;
using namespace ctr::cinb;

// Shapes the tensor-core backward serves; everything else goes to the CUDA-core kernels in cin.cu.
// (internal, not part of the public ABI)
extern "C" __attribute__((visibility("hidden"))) int ctr_cin_bwd_tc_supported(int64_t m, int64_t hk, int64_t D, int64_t H) {
  return m >= 1 && m <= 32 && hk >= 1 && H >= 1 && H <= 128 && (D == 8 || D == 16 || D == 32);
}

extern "C" int64_t ctr_cin_bwd_workspace_bytes(int64_t B, int64_t m, int64_t hk, int64_t D, int64_t H) {
  if (!ctr_cin_bwd_tc_supported(m, hk, D, H)) return 0;
  const int64_t HP = pad_to(H, 32), KRP = (hk + 2) * m + 32;
  return ((2 * KRP + m) * HP + 2 * B * H * D) * (int64_t)sizeof(float);
}

// Returns CTR_OK after enqueueing both tensor-core kernels; the caller has already validated the arguments.
int ctr_cin_bwd_tc(const float* x0, const float* xk, const float* filter, const float* g_out, int64_t B, int64_t m,
                   int64_t hk, int64_t D, int64_t H, float* dx0, float* dxk, float* dfilter, void* workspace,
                   cudaStream_t st) {
  const int HP = (int)pad_to(H, 32), KRP = (int)((hk + 2) * m + 32);
  const int NP = H <= 32 ? 32 : H <= 64 ? 64 : 128;        // wgmma N of the dW kernel
  float* ws_w = static_cast<float*>(workspace);
  float* ws_g = ws_w + (size_t)(2 * KRP + m) * HP;          // + m rows so the i-in-step window of the lo copy stays inside
  {
    const long long total = (long long)KRP * HP;
    split_filter_native_kernel<<<(int)((total + 255) / 256 < 2048 ? (total + 255) / 256 : 2048), 256, 0, st>>>(
        filter, ws_w, (int)(hk * m), (int)H, KRP, HP);
    CTR_CHECK_LAUNCH("ctr_cin_bwd(split filter)");
    const size_t tg = (size_t)B * H * D;
    split_grad_kernel<<<(int)((tg + 255) / 256 < 4096 ? (tg + 255) / 256 : 4096), 256, 0, st>>>(g_out, ws_g, tg);
    CTR_CHECK_LAUNCH("ctr_cin_bwd(split grad)");
  }
  EncodeTiledFn enc = encode_tiled();
  if (enc == nullptr) {
    set_error("ctr_cin_bwd: cuTensorMapEncodeTiled is not available from the driver");
    return CTR_ERR_CUDA;
  }
  int logD = 0;
  while ((1 << logD) < D) ++logD;
  // ---- dX: filter as a 4-D tensor (n_inner 32 | row | i-in-step (stride m rows) | n_outer) so one box lands as
  //      HP/32 K-major [64 rows x 128 B] swizzled sub-tiles holding the rows of i0 and i0+1
  {
    CUtensorMap tmap;
    const cuuint64_t gdim[4] = {32, (cuuint64_t)(2 * KRP), (cuuint64_t)DX_IPS, (cuuint64_t)(HP / 32)};
    const cuuint64_t gstr[3] = {(cuuint64_t)HP * sizeof(float), (cuuint64_t)m * HP * sizeof(float), 32 * sizeof(float)};
    const cuuint32_t box[4] = {32, 32, (cuuint32_t)DX_IPS, (cuuint32_t)(HP / 32)};
    const cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult cr = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, ws_w, gdim, gstr, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("ctr_cin_bwd: cuTensorMapEncodeTiled(filter) failed with CUresult %d", (int)cr);
      return CTR_ERR_CUDA;
    }
    constexpr int SB = 3;
    const int nkb = HP / 32;
    const int smem = SB * 2 * nkb * DX_N * 128 + 8 * 2 * SB + 1024;
    const long long rows = (long long)B * D;
    const int tiles = (int)((rows + DX_TILE - 1) / DX_TILE);
    const int grid = tiles < sm_count() ? tiles : sm_count();
#define DX_LAUNCH(NKB_)                                                                                              \
  {                                                                                                                  \
    auto k = cin_bwd_dx_tc_kernel<SB, NKB_>;                                                                         \
    CTR_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));                            \
    k<<<grid, NTHREADS, smem, st>>>(tmap, x0, xk, g_out, dx0, dxk, (int)B, (int)m, (int)hk, logD, (int)H, KRP);      \
  }
    if (nkb == 1) DX_LAUNCH(1) else if (nkb == 2) DX_LAUNCH(2) else if (nkb == 3) DX_LAUNCH(3) else DX_LAUNCH(4)
#undef DX_LAUNCH
    CTR_CHECK_LAUNCH("ctr_cin_bwd(dx, wgmma)");
  }
  // ---- dW: g (hi | lo stacked along the batch axis) as a 3-D tensor (d | n | b); box = one sample's [NP x D] tile
  //      (rows n >= H are out of bounds and arrive as zeros)
  {
    CUtensorMap tmap;
    const cuuint64_t gdim[3] = {(cuuint64_t)D, (cuuint64_t)H, (cuuint64_t)(2 * B)};
    const cuuint64_t gstr[2] = {(cuuint64_t)D * sizeof(float), (cuuint64_t)H * D * sizeof(float)};
    const cuuint32_t box[3] = {(cuuint32_t)D, (cuuint32_t)NP, 1};
    const cuuint32_t es[3] = {1, 1, 1};
    const CUtensorMapSwizzle sw = D == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : D == 16 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                                                 : CU_TENSOR_MAP_SWIZZLE_32B;
    CUresult cr = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, ws_g, gdim, gstr, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) {
      set_error("ctr_cin_bwd: cuTensorMapEncodeTiled(grad) failed with CUresult %d", (int)cr);
      return CTR_ERR_CUDA;
    }
    const int stage_bytes = 2 * NP * (int)D * 4;
    int sb = (192 * 1024) / stage_bytes;                      // as many stages as 192 KB of shared memory hold, at most 8
    if (sb > 8) sb = 8;
    const int smem = sb * stage_bytes + 8 * 2 * sb + 1024;
    const int ngroups = (int)((hk + DW_IPC - 1) / DW_IPC);
    int nslices = sm_count() / ngroups;
    if (nslices < 1) nslices = 1;
    if (nslices > B) nslices = (int)B;
    const int grid = ngroups * nslices;
    const int chunk = (int)(256 / D);                        // 96 chained MMAs per accumulator before a drain (see cin.cu CHUNK3)
#define DW_LAUNCH(N_, D_)                                                                                            \
  {                                                                                                                  \
    auto k = cin_bwd_dw_tc_kernel<N_, D_>;                                                                           \
    CTR_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));                            \
    k<<<grid, NTHREADS, smem, st>>>(tmap, x0, xk, dfilter, (int)B, (int)m, (int)hk, (int)H, ngroups, nslices, chunk, \
                                    sb);                                                                             \
  }
#define DW_LAUNCH_D(N_)                                                                                              \
  if (D == 8) DW_LAUNCH(N_, 8) else if (D == 16) DW_LAUNCH(N_, 16) else DW_LAUNCH(N_, 32)
    if (NP == 32) { DW_LAUNCH_D(32) } else if (NP == 64) { DW_LAUNCH_D(64) } else { DW_LAUNCH_D(128) }
#undef DW_LAUNCH_D
#undef DW_LAUNCH
    CTR_CHECK_LAUNCH("ctr_cin_bwd(dw, wgmma)");
  }
  return CTR_OK;
}

// AutoInt interacting layer (Song et al., CIKM 2019, arXiv:1810.11921, eq. 5-8): multi-head self-attention over fields.
// The reference tree has no AutoInt code (its README lists AutoInt as a to-do), so the layer follows the paper; parity is
// defined against a float64 restatement of these equations (tests/_autoint_ref.py).
//
//   x (B, F, d); w_query, w_key, w_value, w_res (d, H dk), head h = columns h dk .. h dk + dk - 1; no biases.
//   Q = x Wq, K = x Wk, V = x Wv, R = x Wr                       per sample: F x H dk each
//   A_h = softmax_j(Q_h[i] . K_h[j])                             F x F (no 1/sqrt(dk) scaling: eq. 5-6), row max subtracted
//   O_h = A_h V_h ;  out = relu(concat_h O_h + R)                (B, F, H dk)
// Backward, G = g_out [out > 0]:  dR = dO_h = G_h,  dA = dO V^T,  dV = A^T dO,  dS = A (dA - rowsum(A dA)),
//   dQ = dS K,  dK = dS^T Q,  dx = dQ Wq^T + dK Wk^T + dV Wv^T + dR Wr^T,  dW_p = x^T dP_p.
//
// H100 mapping (csrc/tc_ptx.cuh: wgmma m64nNk8 kind tf32, A in registers, 3xTF32 split, one TMA producer warp).  One
// sample per consumer warpgroup: its F <= 64 fields are the 64 rows of every MMA (zero rows past F).  Each head is padded
// to DKP = 32 or 64 columns and runs as DKP / 32 halves of 32; the weights are prepped once per call into the caller's workspace as tf32 hi | lo copies.
//   autoint_fwd_wgmma_kernel       per head, in 32-column halves: Q_h, K_h, V_h, R_h = x . W^T chunks (the row-chunk GEMMs, x staged in shared
//                                  memory, W^T streamed).  Q_h stays in registers and feeds S = Q_h K_h^T as A fragments;
//                                  K_h is written into a K-major tile.  The softmax runs on the S accumulator; A_h feeds
//                                  O_h = A_h V_h as A fragments, V_h^T reusing the K tile.  R_h is the accumulator O_h starts
//                                  from; out = relu(.) is the only global write.  Q, K, V, R and S never leave the SM.
//   autoint_bwd_attn_wgmma_kernel  recomputes Q_h, K_h and A_h as the forward does and leaves A_h in a [64][TP] shared
//                                  buffer.  Then dV = A^T dO (A^T read from the buffer), V_h, dA = dO V_h^T on the fragment
//                                  path, and dS = A (dA - rowsum(A dA)) written over A in the buffer; dQ = dS K_h and
//                                  dK = dS^T Q_h read dS from it.  K_h and Q_h are projected a second time as the B
//                                  operands of those two GEMMs, so no score-sized array stays in registers across a GEMM.
//                                  Writes dP = dQ | dK | dV | dR (B F, 4 H dk) to the workspace.
//   autoint_bwd_dx_wgmma_kernel    dx = dP . [Wq; Wk; Wv; Wr]^T: dP rows loaded straight into accumulator-layout A fragments,
//                                  the weights streamed as a hidden operand (perm8 order, tc_ptx.cuh rows::).
//   dW                             dW_p = x^T dP_p over the B F rows: tc_ptx.cuh's weight_grad_wgmma_kernel (DwRows).
// Rows of x, out and g_out are d or H dk floats (not 16-byte multiples in general), so they move with ordinary loads.
//
// Bounds: 1 <= F <= 64, 1 <= d <= 128, 1 <= dk <= 64, 1 <= H <= 8, H dk <= 128, B >= 0; CTR_ERR_UNSUPPORTED otherwise.
#include "tc_ptx.cuh"

namespace ctr {
namespace autoint {
using namespace ctr::tc;
using namespace ctr::tc::rows;

constexpr int FP = 64;                       // fields per sample tile: the M of every MMA, the N / K of the attention GEMMs
constexpr int TP = FP + 8;                   // pitch of the transpose buffer: conflict-free transposed A-fragment reads

struct W4 {
  const float* p[4];                         // w_query, w_key, w_value, w_res (d, HD)
};

// position of column u inside its group of 8 in a B tile fed by rows::acc_to_a fragments (the inverse of perm8)
__device__ __forceinline__ int pos8(int u) { return (u & ~7) | ((u & 7) >> 1) | ((u & 1) << 2); }

// mode 0: the forward / recompute operand, W^T headwise [RU = 4 H DKP units][DP], unit (h 4 + p) DKP + c = W_p[:, h dk + c];
// mode 1: the dx operand, W [DP][UP] natural order (unit p HD + col), units perm8 within each group of 8.
__global__ void autoint_prep_kernel(W4 w, float* __restrict__ dst, int d, int H, int dk, int DP, int DKP, int UP, int mode) {
  const int HD = H * dk;
  const size_t total = mode == 0 ? (size_t)4 * H * DKP * DP : (size_t)DP * UP;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    int i, p, col;
    bool in;
    if (mode == 0) {
      const int u = (int)(idx / DP), c = u % DKP, hp = u / DKP;
      i = (int)(idx % DP); p = hp & 3; col = (hp >> 2) * dk + c; in = c < dk;
    } else {
      const int u = perm8((int)(idx % UP));
      i = (int)(idx / UP); p = u / HD; col = u % HD; in = u < 4 * HD;
    }
    const float* src = p == 0 ? w.p[0] : p == 1 ? w.p[1] : p == 2 ? w.p[2] : w.p[3];
    const float v = (in && i < d) ? __ldg(src + (size_t)i * HD + col) : 0.f;
    store_split(dst, total, idx, v);
  }
}

// ---------------------------------------------------------------------------------------------- attention tiles
// A K-layout tile holds a [64 rows x KP] operand as KP / 32 blocks of [64 x 32] (hi | lo), column u at pos8(u);
// a T-layout tile holds the transpose of a [64 rows x NR] operand as 2 blocks of [NR x 32 rows] (hi | lo).
template <int KP>
__device__ __forceinline__ void store_klayout(float* tile, const float (&a)[HC / 2], int kb, int r0, int t) {
  float* blk = tile + kb * (FP * KB * 2);
#pragma unroll
  for (int q = 0; q < HC / 2; ++q) {
    const int u = 8 * (q >> 2) + 2 * t + (q & 1), r = r0 + 8 * ((q >> 1) & 1);
    store_split_sw128(blk, FP, r, pos8(u), a[q]);
  }
}
template <int NR>
__device__ __forceinline__ void store_tlayout(float* tile, int r, int u, float v, bool perm) {
  store_split_sw128(tile + (r / KB) * (NR * KB * 2), NR, u, perm ? pos8(r % KB) : r % KB, v);
}
// the accumulator [64 x 32 columns kb 32 ..] of this thread into a T-layout tile of NR rows
template <int NR>
__device__ __forceinline__ void store_tlayout_acc(float* tile, const float (&a)[HC / 2], int kb, int r0, int t, bool perm) {
#pragma unroll
  for (int q = 0; q < HC / 2; ++q)
    store_tlayout<NR>(tile, r0 + 8 * ((q >> 1) & 1), kb * HC + 8 * (q >> 2) + 2 * t + (q & 1), a[q], perm);
}

// D[64 x N] (+)= A[64 x KP] . B: A from this thread's accumulator-layout registers a (KP / 2 floats, acc_to_a order), B a
// tile of KP / 32 blocks [N x 32] (hi | lo) with columns at pos8.  k-steps at or past nk are skipped (zero columns);
// accumulate == false starts from zero.
template <int N, int KP>
__device__ __forceinline__ void gemm_acc_a(float (&d)[N / 2], const float (&a)[KP / 2], uint32_t tile, int nk,
                                           bool accumulate) {
#pragma unroll
  for (int kb = 0; kb < KP / KB; ++kb) {
    if (4 * kb >= nk) break;
    float v[HC / 2];
#pragma unroll
    for (int q = 0; q < HC / 2; ++q) v[q] = a[kb * (HC / 2) + q];
    uint32_t ah[4][4], al[4][4];
    acc_to_a(v, ah, al);
    const uint32_t blk = tile + kb * (N * 128 * 2);
    const uint64_t bhi = gmma_desc_kmajor(blk, 128), blo = gmma_desc_kmajor(blk + N * 128, 128);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      if (4 * kb + ks < nk) mma_3xtf32<N>(d, ah[ks], al[ks], bhi, blo, 2 * ks, (accumulate || kb || ks) ? 1 : 0);
    wgmma_commit();
    wgmma_wait_keep(ah, al);
  }
}
// D[64 x N] = A[64 x 64] . B with A read from a [64][TP] shared-memory buffer: A[m][k] = T[k TP + m] (TRANS) or
// T[m TP + k]; B a T-layout tile of N rows (natural k).
template <int N, bool TRANS>
__device__ __forceinline__ void gemm_buf_a(float (&d)[N / 2], const float* T, int r0, int t, uint32_t tile, int nk) {
#pragma unroll
  for (int kb = 0; kb < FP / KB; ++kb) {
    if (4 * kb >= nk) break;
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      float a[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int k = kb * KB + 8 * ks + t + 4 * (q >> 1), m = r0 + 8 * (q & 1);
        a[q] = TRANS ? T[k * TP + m] : T[m * TP + k];
      }
      tf32_split(a, ah[ks], al[ks]);
    }
    const uint32_t blk = tile + kb * (N * 128 * 2);
    const uint64_t bhi = gmma_desc_kmajor(blk, 128), blo = gmma_desc_kmajor(blk + N * 128, 128);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      if (4 * kb + ks < nk) mma_3xtf32<N>(d, ah[ks], al[ks], bhi, blo, 2 * ks, (kb || ks) ? 1 : 0);
    wgmma_commit();
    wgmma_wait_keep(ah, al);
  }
}

// Row softmax of the score accumulator (rows r0, r0 + 8; columns 8c + 2t + e spread over the 4 threads of a quad), columns
// at or past F masked out.
__device__ __forceinline__ void softmax_rows(float (&s)[FP / 2], int F, int t) {
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float m = -INFINITY;
#pragma unroll
    for (int c = 0; c < FP / 8; ++c)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& v = s[4 * c + 2 * r + e];
        if (8 * c + 2 * t + e >= F) v = -INFINITY;
        m = fmaxf(m, v);
      }
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    float l = 0.f;
#pragma unroll
    for (int c = 0; c < FP / 8; ++c)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float& v = s[4 * c + 2 * r + e];
        v = expf(v - m);
        l += v;
      }
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.f / l;
#pragma unroll
    for (int c = 0; c < FP / 8; ++c)
#pragma unroll
      for (int e = 0; e < 2; ++e) s[4 * c + 2 * r + e] *= inv;
  }
}

// fixed shared memory of the attention kernels next to their ring (1 KB alignment slack included), and the ring depth
__host__ __device__ constexpr int fwd_fixed_bytes(int DP, int DKP) {
  return NWG * (FP * HC * 8 + WG_M * row_pitch(DP) * 4) + 64 + 1024;
}
__host__ __device__ constexpr int bwd_fixed_bytes(int DP) {
  return NWG * (FP * HC * 8 + WG_M * row_pitch(DP) * 4 + FP * TP * 4) + 64 + 1024;
}
__host__ __device__ constexpr int ring_depth(int fixed, int DP) {
  return (int)((SMEM_CAP - fixed) / stage_bytes(DP)) < 4 ? (int)((SMEM_CAP - fixed) / stage_bytes(DP)) : 4;
}

// S = sum over the head's 32-column halves of Q_hf K_hf^T, the Q and K chunks of each half taken from the ring in turn:
// Q_hf stays in registers (A fragments), K_hf goes through the warpgroup's K-layout tile.  Returns with the tile free.
template <int DP>
__device__ __forceinline__ void score_halves(float (&s)[FP / 2], Ring& ring, const float* xw, float* kv, uint32_t kv_u,
                                             uint32_t sbase, int r0, int t, int lane, int wg, int dk, int nkb) {
  constexpr int SBYTES = stage_bytes(DP);
#pragma unroll 1
  for (int hf = 0; hf < nkb; ++hf) {
    float qa[HC / 2], a[HC / 2];
    gemm_rows<DP>(qa, xw, r0, t, sbase + ring.wait() * SBYTES);
    ring.release(lane);
    gemm_rows<DP>(a, xw, r0, t, sbase + ring.wait() * SBYTES);
    ring.release(lane);
    store_klayout<HC>(kv, a, 0, r0, t);
    fence_proxy_async();
    wg_bar_sync(1 + wg);
    gemm_acc_a<FP, HC>(s, qa, kv_u, min(4, (dk - HC * hf + 7) / 8), hf > 0);
    wg_bar_sync(1 + wg);                      // K_hf reads retired
  }
}

// ================================================================================================= forward
template <int DP, int DKP, int SB>
__global__ void __launch_bounds__(NTHREADS, 1)
autoint_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_wt, const float* __restrict__ x, float* __restrict__ out,
                         int B, int F, int d, int H, int dk) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int SBYTES = stage_bytes(DP), LD = row_pitch(DP), NKB = DKP / HC, TILE_F = FP * HC * 2;
  float* tiles = reinterpret_cast<float*>(smem + SB * SBYTES);             // [2][FP HC 2]  K_h, then V_h^T halves
  float* xs = tiles + NWG * TILE_F;                                         // [2][64][LD]
  const uint32_t sbase = smem_u32(smem);
  Ring ring(smem_u32(xs + NWG * WG_M * LD), SB);
  const int RU = 4 * H * DKP, HD = H * dk;

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_tiles = (B + NWG - 1) / NWG;
  ring.init();
  // ============================ TMA producer: per head and 32-column half, W^T chunks Q, K ..., then V, R ... ======
  if (producer_role(warp, lane, [&] {
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x)
          for (int h = 0; h < H; ++h)
            for (int j = 0; j < 4 * NKB; ++j) {
              const int p = (j % 2) + (j < 2 * NKB ? 0 : 2), hf = (j % (2 * NKB)) / 2;
              const Ring::Slot slot = ring.acquire(SBYTES);
              load_rows_operand<DP>(sbase + slot.stage * SBYTES, &tmap_wt, (h * 4 + p) * NKB + hf, RU, slot.full);
            }
      }))
    return;

  // ============================ consumers: one sample per warpgroup ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3, tw = threadIdx.x & 127;
  const int r0 = w * 16 + g;
  float* xw = xs + wg * WG_M * LD;
  float* kv = tiles + wg * TILE_F;
  const uint32_t kv_u = smem_u32(kv);
  const int nk_f = (F + 7) / 8;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long b = (long long)tile * NWG + wg;
    const long long row0 = b * F;
    stage_rows<DP>(xw, x, nullptr, row0, b < B ? (int)(row0 + F) : 0, d, tw);
    wg_bar_sync(1 + wg);
    for (int h = 0; h < H; ++h) {
      float s[FP / 2];
      score_halves<DP>(s, ring, xw, kv, kv_u, sbase, r0, t, lane, wg, dk, NKB);
      softmax_rows(s, F, t);
#pragma unroll
      for (int hf = 0; hf < NKB; ++hf) {      // per 32-column half: V_h^T into the tile, O = R + A V
        float a[HC / 2];
        gemm_rows<DP>(a, xw, r0, t, sbase + ring.wait() * SBYTES);
        ring.release(lane);
        store_tlayout_acc<HC>(kv, a, 0, r0, t, true);
        fence_proxy_async();
        wg_bar_sync(1 + wg);
        float o[HC / 2];
        gemm_rows<DP>(o, xw, r0, t, sbase + ring.wait() * SBYTES);
        ring.release(lane);
        gemm_acc_a<HC, FP>(o, s, kv_u, nk_f, true);
        if (b < B) {
#pragma unroll
          for (int q = 0; q < HC / 2; ++q) {
            const int u = HC * hf + 8 * (q >> 2) + 2 * t + (q & 1), r = r0 + 8 * ((q >> 1) & 1);
            if (u < dk && r < F) out[(size_t)(row0 + r) * HD + h * dk + u] = fmaxf(o[q], 0.f);
          }
        }
        wg_bar_sync(1 + wg);                  // V_h^T reads retired before the tile is rewritten
      }
    }
  }
}

// ================================================================================================= backward: attention
// a [64 x 64] accumulator of this thread into the row-major transpose buffer
__device__ __forceinline__ void store_acc_rows(float* T, const float (&a)[FP / 2], int r0, int t) {
#pragma unroll
  for (int q = 0; q < FP / 2; ++q) T[(r0 + 8 * ((q >> 1) & 1)) * TP + 8 * (q >> 2) + 2 * t + (q & 1)] = a[q];
}

// per-row projection gradients dP (rows B F, 4 HD): projection p, head h, column u -> p HD + h dk + u
template <int N>
__device__ __forceinline__ void stage_dp(float* __restrict__ dp, const float (&a)[N], long long row0, int F, int HD, int col0,
                                         int dk, int r0, int t, bool live) {
  if (!live) return;
#pragma unroll
  for (int q = 0; q < N; ++q) {
    const int u = 8 * (q >> 2) + 2 * t + (q & 1), r = r0 + 8 * ((q >> 1) & 1);
    if (u < dk && r < F) dp[(size_t)(row0 + r) * (4 * HD) + col0 + u] = a[q];
  }
}

// NKB = DKP / 32 is a run-time argument here: the 32-column halves run as rolled loops whatever the head width
template <int DP, int SB>
__global__ void __launch_bounds__(NTHREADS, 1)
autoint_bwd_attn_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_wt, const float* __restrict__ x,
                              const float* __restrict__ outv, const float* __restrict__ g_out, float* __restrict__ dp,
                              int B, int F, int d, int H, int dk, int NKB) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int SBYTES = stage_bytes(DP), LD = row_pitch(DP), TILE_F = FP * HC * 2;
  float* tiles = reinterpret_cast<float*>(smem + SB * SBYTES);             // [2][FP HC 2]  the operand tile
  float* xs = tiles + NWG * TILE_F;                                         // [2][64][LD]
  float* ts = xs + NWG * WG_M * LD;                                         // [2][64][TP]  A, then dS in place
  const uint32_t sbase = smem_u32(smem);
  Ring ring(smem_u32(ts + NWG * FP * TP), SB);
  const int RU = 4 * H * NKB * HC, HD = H * dk;

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_tiles = (B + NWG - 1) / NWG;
  ring.init();
  // ============================ TMA producer: per head, the W^T chunks of Q, K, V, K, Q ===========================
  if (producer_role(warp, lane, [&] {
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x)
          for (int h = 0; h < H; ++h)
            for (int j = 0; j < 5 * NKB; ++j) {       // per half Q, K; then per half V, then K, then Q again
              int p, hf;
              if (j < 2 * NKB) { p = j % 2; hf = j / 2; }
              else { p = 2 - (j - 2 * NKB) / NKB; hf = (j - 2 * NKB) % NKB; }
              const Ring::Slot slot = ring.acquire(SBYTES);
              load_rows_operand<DP>(sbase + slot.stage * SBYTES, &tmap_wt, (h * 4 + p) * NKB + hf, RU, slot.full);
            }
      }))
    return;

  // ============================ consumers: one sample per warpgroup ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3, tw = threadIdx.x & 127;
  const int r0 = w * 16 + g;
  float* xw = xs + wg * WG_M * LD;
  float* kv = tiles + wg * TILE_F;
  float* T = ts + wg * FP * TP;
  const uint32_t kv_u = smem_u32(kv);
  const int nk_f = (F + 7) / 8;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long b = (long long)tile * NWG + wg;
    const long long row0 = b * F;
    const bool live = b < B;
    stage_rows<DP>(xw, x, nullptr, row0, live ? (int)(row0 + F) : 0, d, tw);
    wg_bar_sync(1 + wg);
    for (int h = 0; h < H; ++h) {
      // ---- recompute A_h into T
      {
        float p[FP / 2];
        score_halves<DP>(p, ring, xw, kv, kv_u, sbase, r0, t, lane, wg, dk, NKB);
        softmax_rows(p, F, t);
        store_acc_rows(T, p, r0, t);
      }
      wg_bar_sync(1 + wg);                    // A visible in T
      // ---- per half: dV = A^T dO (A^T from T, dO^T into the tile)
#pragma unroll 1
      for (int hf = 0; hf < NKB; ++hf) {
        for (int idx = tw; idx < FP * HC; idx += 128) {
          const int i = idx / HC, u = idx % HC;
          float v = 0.f;
          if (live && HC * hf + u < dk && i < F) {
            const size_t o = (size_t)(row0 + i) * HD + h * dk + HC * hf + u;
            v = __ldg(outv + o) > 0.f ? __ldg(g_out + o) : 0.f;
          }
          store_tlayout<HC>(kv, i, u, v, false);
        }
        fence_proxy_async();
        wg_bar_sync(1 + wg);
        float dv[HC / 2];
        gemm_buf_a<HC, true>(dv, T, r0, t, kv_u, nk_f);
        stage_dp(dp, dv, row0, F, HD, 2 * HD + h * dk + HC * hf, dk - HC * hf, r0, t, live);
        wg_bar_sync(1 + wg);                  // dO^T reads retired
      }
      // ---- dA = sum over halves of dO V_h^T (V_h half in the K-layout tile), dO = G_h (it is also dR);
      //      dS = A (dA - rowsum(A dA)) written over A in T
      {
        float ds[FP / 2];
#pragma unroll 1
        for (int hf = 0; hf < NKB; ++hf) {
          float a[HC / 2];
          gemm_rows<DP>(a, xw, r0, t, sbase + ring.wait() * SBYTES);
          ring.release(lane);
          store_klayout<HC>(kv, a, 0, r0, t);
          fence_proxy_async();
          wg_bar_sync(1 + wg);
          float go[HC / 2];
#pragma unroll
          for (int q = 0; q < HC / 2; ++q) {
            const int u = HC * hf + 8 * (q >> 2) + 2 * t + (q & 1), r = r0 + 8 * ((q >> 1) & 1);
            float v = 0.f;
            if (live && u < dk && r < F) {
              const size_t o = (size_t)(row0 + r) * HD + h * dk + u;
              v = __ldg(outv + o) > 0.f ? __ldg(g_out + o) : 0.f;
            }
            go[q] = v;
          }
          stage_dp(dp, go, row0, F, HD, 3 * HD + h * dk + HC * hf, dk - HC * hf, r0, t, live);
          gemm_acc_a<FP, HC>(ds, go, kv_u, min(4, (dk - HC * hf + 7) / 8), hf > 0);
          wg_bar_sync(1 + wg);                // V_h reads retired
        }
        // each thread reads and overwrites only its own entries of T
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float dsum = 0.f;
#pragma unroll
          for (int c = 0; c < FP / 8; ++c)
#pragma unroll
            for (int e = 0; e < 2; ++e) dsum += T[(r0 + 8 * r) * TP + 8 * c + 2 * t + e] * ds[4 * c + 2 * r + e];
          dsum += __shfl_xor_sync(0xffffffffu, dsum, 1);
          dsum += __shfl_xor_sync(0xffffffffu, dsum, 2);
#pragma unroll
          for (int c = 0; c < FP / 8; ++c)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float& a = T[(r0 + 8 * r) * TP + 8 * c + 2 * t + e];
              a = a * (ds[4 * c + 2 * r + e] - dsum);
            }
        }
      }
      wg_bar_sync(1 + wg);                    // dS visible in T
      // ---- per half: dQ = dS K_h (K_h recomputed as K_h^T), then dK = dS^T Q_h (Q_h recomputed as Q_h^T)
#pragma unroll 1
      for (int hf = 0; hf < NKB; ++hf) {
        float a[HC / 2];
        gemm_rows<DP>(a, xw, r0, t, sbase + ring.wait() * SBYTES);
        ring.release(lane);
        store_tlayout_acc<HC>(kv, a, 0, r0, t, false);
        fence_proxy_async();
        wg_bar_sync(1 + wg);
        gemm_buf_a<HC, false>(a, T, r0, t, kv_u, nk_f);
        stage_dp(dp, a, row0, F, HD, h * dk + HC * hf, dk - HC * hf, r0, t, live);
        wg_bar_sync(1 + wg);                  // K_h^T reads retired
      }
#pragma unroll 1
      for (int hf = 0; hf < NKB; ++hf) {
        float a[HC / 2];
        gemm_rows<DP>(a, xw, r0, t, sbase + ring.wait() * SBYTES);
        ring.release(lane);
        store_tlayout_acc<HC>(kv, a, 0, r0, t, false);
        fence_proxy_async();
        wg_bar_sync(1 + wg);
        gemm_buf_a<HC, true>(a, T, r0, t, kv_u, nk_f);
        stage_dp(dp, a, row0, F, HD, HD + h * dk + HC * hf, dk - HC * hf, r0, t, live);
        wg_bar_sync(1 + wg);                  // Q_h^T reads retired
      }
    }
  }
}

// ================================================================================================= backward: dx
constexpr int DX_TILE = NWG * WG_M;          // rows (sample fields) per CTA tile

template <int DP, int SB>
__global__ void __launch_bounds__(NTHREADS, 1)
autoint_bwd_dx_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_w, const float* __restrict__ dp,
                            float* __restrict__ d_x, int rows_total, int d, int U, int UP) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int SBYTES = stage_bytes(DP);
  const uint32_t sbase = smem_u32(smem);
  Ring ring(sbase + SB * SBYTES, SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_tiles = (rows_total + DX_TILE - 1) / DX_TILE, NC = UP / HC;
  ring.init();
  if (producer_role(warp, lane, [&] {
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x)
          for (int j = 0; j < NC; ++j) {
            const Ring::Slot slot = ring.acquire(SBYTES);
            load_hidden_operand<DP>(sbase + slot.stage * SBYTES, &tmap_w, j, slot.full);
          }
      }))
    return;

  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3;
  const int r0 = w * 16 + g;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long base = (long long)tile * DX_TILE + wg * WG_M;
    const bool v0 = base + r0 < rows_total, v1 = base + r0 + 8 < rows_total;
    const float* p0 = dp + (size_t)(base + r0) * U;
    float acc[DP / 2], dacc[DP / 2];
#pragma unroll
    for (int q = 0; q < DP / 2; ++q) { acc[q] = 0.f; dacc[q] = 0.f; }
    for (int j = 0; j < NC; ++j) {
      float a[HC / 2];
#pragma unroll
      for (int q = 0; q < HC / 2; ++q) {
        const int col = j * HC + 8 * (q >> 2) + 2 * t + (q & 1);
        const bool hi = (q >> 1) & 1;
        a[q] = (col < U && (hi ? v1 : v0)) ? __ldg(p0 + (hi ? (size_t)8 * U : 0) + col) : 0.f;
      }
      uint32_t hh[HC / 8][4], hl[HC / 8][4];
      acc_to_a(a, hh, hl);
      gemm_hidden<DP>(dacc, hh, hl, sbase + ring.wait() * SBYTES, chain_first(j, CHAIN));
      ring.release(lane);
      if (chain_last(j, NC, CHAIN)) chain_drain(acc, dacc);
    }
#pragma unroll
    for (int c = 0; c < DP / 8; ++c)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int i = 8 * c + 2 * t + e;
        if (i < d) {
          if (v0) d_x[(size_t)(base + r0) * d + i] = acc[4 * c + e];
          if (v1) d_x[(size_t)(base + r0 + 8) * d + i] = acc[4 * c + 2 + e];
        }
      }
  }
}

// ================================================================================================= backward: dW
// Result rows of tc::weight_grad_wgmma_kernel over P = dP (B F, 4 HD), Q = x: row u is dW_p[:, u % HD] with p = u / HD.
struct DwRows {
  static constexpr bool row_sums = false, mask_q = false, slice_d = false;
  float* dw[4];                              // d_w_query, d_w_key, d_w_value, d_w_res (d, HD)
  int HD;
  __device__ __forceinline__ GradRow row(int u) const {
    if (u >= 4 * HD) return GradRow{};
    const int p = u / HD;
    float* dst = p == 0 ? dw[0] : p == 1 ? dw[1] : p == 2 ? dw[2] : dw[3];
    return GradRow{dst + u % HD, HD};
  }
};

}  // namespace autoint
}  // namespace ctr

// ------------------------------------------------------------------------------------------------ host
using namespace ctr;
using namespace ctr::autoint;

namespace {

struct AiShape {
  int DP, DKP;
  int64_t RU, UP, U;               // headwise units (4 H DKP), natural units padded to 32 (dx operand), natural units 4 H dk
  int64_t wt_floats, w_floats;     // prepped operands: W^T headwise [2 RU][DP], W natural [2 DP][UP]
  int64_t w_offset, dp_offset;     // workspace byte offsets of W natural and dP (B F, U) (backward)
  int64_t fwd_bytes, bwd_bytes;
};

AiShape shape_of(int64_t B, int64_t F, int64_t d, int64_t H, int64_t dk) {
  AiShape s;
  s.DP = dp_class(d);
  s.DKP = dk <= 32 ? 32 : 64;
  s.RU = 4 * H * s.DKP;
  s.U = 4 * H * dk;
  s.UP = pad_to(s.U, HC);
  s.wt_floats = 2 * s.RU * s.DP;
  s.w_floats = 2 * s.DP * s.UP;
  s.fwd_bytes = pad_to(s.wt_floats * (int64_t)sizeof(float), 128);
  s.w_offset = s.fwd_bytes;
  s.dp_offset = s.w_offset + pad_to(s.w_floats * (int64_t)sizeof(float), 128);
  s.bwd_bytes = s.dp_offset + pad_to(B * F * s.U * (int64_t)sizeof(float), 128);
  return s;
}

int check_shape(const char* fn, int64_t B, int64_t F, int64_t d, int64_t H, int64_t dk) {
  CTR_REQUIRE(B >= 0 && F >= 1 && d >= 1 && H >= 1 && dk >= 1, "%s: bad sizes B=%lld F=%lld d=%lld H=%lld dk=%lld", fn,
              (long long)B, (long long)F, (long long)d, (long long)H, (long long)dk);
  CTR_UNSUPPORTED(F > 64, "%s: unsupported field count F=%lld (the kernels take F <= 64)", fn, (long long)F);
  CTR_UNSUPPORTED(d > 128, "%s: unsupported input width d=%lld (the kernels take d <= 128)", fn, (long long)d);
  CTR_UNSUPPORTED(dk > 64, "%s: unsupported head width dk=%lld (the kernels take dk <= 64)", fn, (long long)dk);
  CTR_UNSUPPORTED(H > 8, "%s: unsupported head count H=%lld (the kernels take H <= 8)", fn, (long long)H);
  CTR_UNSUPPORTED(H * dk > 128, "%s: unsupported output width H*dk=%lld (the kernels take H*dk <= 128)", fn,
                  (long long)(H * dk));
  CTR_UNSUPPORTED(B * F > 0x7fffff00LL, "%s: batch too large (B*F=%lld)", fn, (long long)(B * F));
  return CTR_OK;
}

int prep(const char* what, const W4& w, float* dst, int64_t d, int64_t H, int64_t dk, const AiShape& s, int mode,
         cudaStream_t st) {
  const int64_t total = mode == 0 ? s.RU * s.DP : s.DP * s.UP;
  return launch(what, autoint_prep_kernel, dim3(capped_grid((total + 255) / 256, 1024)), 256, 0, st, w, dst, (int)d, (int)H,
                (int)dk, s.DP, s.DKP, (int)s.UP, mode);
}

template <class F>
int with_shape(const AiShape& s, F&& f) {
  return with_const<32, 64, 96, 128>(s.DP, [&](auto DP) {
    return with_const<32, 64>(s.DKP, [&](auto DKP) { return f(DP, DKP); });
  });
}

}  // namespace

extern "C" int ctr_autoint_workspace_bytes(int64_t B, int64_t F, int64_t d, int64_t H, int64_t dk, int64_t* bytes) {
  int rc = check_shape("ctr_autoint_workspace_bytes", B, F, d, H, dk);
  if (rc) return rc;
  CTR_REQUIRE(bytes != nullptr, "ctr_autoint_workspace_bytes: null argument");
  *bytes = shape_of(B, F, d, H, dk).bwd_bytes;
  return CTR_OK;
}

extern "C" int ctr_autoint_fwd(const float* x, const float* w_query, const float* w_key, const float* w_value,
                               const float* w_res, int64_t B, int64_t F, int64_t d, int64_t H, int64_t dk, float* out,
                               void* workspace, int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_autoint_fwd";
  int rc = check_shape(fn, B, F, d, H, dk);
  if (rc) return rc;
  CTR_REQUIRE(x && w_query && w_key && w_value && w_res && out, "ctr_autoint_fwd: null argument");
  const AiShape s = shape_of(B, F, d, H, dk);
  rc = check_workspace(fn, "ctr_autoint_workspace_bytes with B = 0", workspace, workspace_bytes, s.fwd_bytes);
  if (rc) return rc;
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  float* ws = static_cast<float*>(workspace);
  const W4 w = {{w_query, w_key, w_value, w_res}};
  if ((rc = prep("ctr_autoint_fwd(prep)", w, ws, d, H, dk, s, 0, st))) return rc;
  CUtensorMap mwt;
  if ((rc = encode_rows_operand(fn, &mwt, ws, s.DP, s.RU))) return rc;
  const int grid = capped_grid((B + NWG - 1) / NWG, sm_count());
  return with_shape(s, [&](auto DP, auto DKP) {
    constexpr int SB = ring_depth(fwd_fixed_bytes(DP, DKP), DP);
    static_assert(SB >= 1, "forward shared memory");
    const size_t smem = fwd_fixed_bytes(DP, DKP) - 64 + 16 * SB + SB * stage_bytes(DP);
    return launch("ctr_autoint_fwd(wgmma)", autoint_fwd_wgmma_kernel<DP, DKP, SB>, grid, NTHREADS, smem, st, mwt, x, out,
                  (int)B, (int)F, (int)d, (int)H, (int)dk);
  });
}

extern "C" int ctr_autoint_bwd(const float* x, const float* w_query, const float* w_key, const float* w_value,
                               const float* w_res, const float* out, const float* g_out, int64_t B, int64_t F, int64_t d,
                               int64_t H, int64_t dk, float* d_x, float* d_w_query, float* d_w_key, float* d_w_value,
                               float* d_w_res, void* workspace, int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_autoint_bwd";
  int rc = check_shape(fn, B, F, d, H, dk);
  if (rc) return rc;
  CTR_REQUIRE(x && w_query && w_key && w_value && w_res && out && g_out && d_x && d_w_query && d_w_key && d_w_value &&
                  d_w_res,
              "ctr_autoint_bwd: null argument");
  const AiShape s = shape_of(B, F, d, H, dk);
  rc = check_workspace(fn, "ctr_autoint_workspace_bytes", workspace, workspace_bytes, s.bwd_bytes);
  if (rc) return rc;
  cudaStream_t st = as_stream(stream);
  const size_t wbytes = sizeof(float) * (size_t)(d * H * dk);
  for (float* p : {d_w_query, d_w_key, d_w_value, d_w_res}) CTR_CUDA(cudaMemsetAsync(p, 0, wbytes, st));
  if (B == 0) return CTR_OK;
  float* ws = static_cast<float*>(workspace);
  float* wn = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + s.w_offset);
  float* dp = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + s.dp_offset);
  const W4 w = {{w_query, w_key, w_value, w_res}};
  if ((rc = prep("ctr_autoint_bwd(prep)", w, ws, d, H, dk, s, 0, st)) ||
      (rc = prep("ctr_autoint_bwd(prep)", w, wn, d, H, dk, s, 1, st)))
    return rc;
  const int64_t rows = B * F;
  CUtensorMap mwt, mw;
  if ((rc = encode_rows_operand(fn, &mwt, ws, s.DP, s.RU)) || (rc = encode_hidden_operand(fn, &mw, wn, s.DP, s.UP)))
    return rc;
  const int sms = sm_count();
  const DwRows dw = {{d_w_query, d_w_key, d_w_value, d_w_res}, (int)(H * dk)};
  rc = with_const<32, 64, 96, 128>(s.DP, [&](auto DP) {
    constexpr int SB = ring_depth(bwd_fixed_bytes(DP), DP);
    static_assert(SB >= 2, "attention backward shared memory");
    const size_t smem = bwd_fixed_bytes(DP) - 64 + 16 * SB + SB * stage_bytes(DP);
    return launch("ctr_autoint_bwd(attention, wgmma)", autoint_bwd_attn_wgmma_kernel<DP, SB>,
                  capped_grid((B + NWG - 1) / NWG, sms), NTHREADS, smem, st, mwt, x, out, g_out, dp, (int)B, (int)F, (int)d,
                  (int)H, (int)dk, s.DKP / HC);
  });
  if (rc) return rc;
  // dx and dW read the natural-order dP: one instantiation per input width
  return with_const<32, 64, 96, 128>(s.DP, [&](auto DP) {
    constexpr int SBX = 4;
    static_assert(SBX * (stage_bytes(DP) + 16) + 1024 <= SMEM_CAP, "dx shared memory");
    if (int r = launch("ctr_autoint_bwd(dx, wgmma)", autoint_bwd_dx_wgmma_kernel<DP, SBX>,
                       capped_grid((rows + DX_TILE - 1) / DX_TILE, sms), NTHREADS, SBX * (stage_bytes(DP) + 16) + 1024, st,
                       mw, dp, d_x, (int)rows, (int)d, (int)s.U, (int)s.UP))
      return r;
    return launch_weight_grad<DP>(fn, "ctr_autoint_bwd(dw, wgmma)", dw, dp, s.U, rows, x, nullptr, (int)d, 1, st);
  });
}

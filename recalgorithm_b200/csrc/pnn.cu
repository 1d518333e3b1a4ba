// PNN product layer (IPNN / OPNN) -- PNN/pnn.py:125-181.
//
//   lz[b,n]  = sum_i e_flat[b,i] linear_w[i,n]                                      (:133-139)
//   IPNN     lp[b,n] = sum_k (sum_f theta[n,f] e[b,f,k])^2                          (:146-158)
//   OPNN     lp[b,n] = sum_kl s[b,k] s[b,l] W_n[min(k,l), max(k,l)],  s = sum_f e_f (:160-173)
//   out      = relu(lz + lp + bias)                                                  (:181)
//
// Both product methods are linear maps of a small per-sample quadratic feature vector, so the whole layer is one GEMM
//   out[b,:] = relu(xt_b . Wm),   xt_b = [e_flat (FK) | q (Q) | 1],   Wm = [linear_w ; product weights ; bias]  (WX x N)
// with, for pairs i <= j in row-major upper-triangle order and c = 1 on the diagonal, 2 off it:
//   IPNN  q_ij = <e_i, e_j>  (Q = F(F+1)/2),  Wm[FK + q(i,j), n] = c theta[n,i] theta[n,j]
//   OPNN  q_kl = s_k s_l     (Q = K(K+1)/2),  Wm[FK + q(k,l), n] = c W_n[k,l]        (the lower triangle never enters)
// Wm is derived from the variables once per call (prep kernel).  The backward is two GEMMs with G = g_out * [out > 0]:
//   dxt  = G . Wm^T       (per sample; the chain rule through q turns it into d_e)
//   dWm^T = G^T . xt      (over the batch; the fold kernel turns it into d_linear_w, d_product_w and d_bias)
//
// H100 mapping (the CIN kernels' pattern, csrc/tc_ptx.cuh): two consumer warpgroups of 64 rows + one TMA producer warp,
// wgmma m64nNk8 kind tf32 with the generated operand in registers, 3xTF32 split for fp32-class accuracy, fp32 accumulators
// drained every 96 chained MMAs, every output overwritten.
//   pnn_fwd_tc_kernel     A = xt (rows = samples), formed once per tile from the staged e rows and reused over the N loop;
//                         B = Wm^T [64 n x WP] tiles (TMA, SWIZZLE_128B).  Epilogue: relu, stores.
//   pnn_bwd_dx_tc_kernel  A = G (rows = samples, K = n), formed per 32-column block from g_out and out;
//                         B = Wm [WP x 32 n] tiles (TMA).  Epilogue: dxt -> shared memory -> chain rule -> d_e.
//   pnn_bwd_dw_tc_kernel  A = G^T (rows = n, K = samples) from TMA-staged g_out / out chunks of 32 samples;
//                         B = xt^T [WP x 32 samples], generated on chip into 128B-swizzled shared memory.
//                         A CTA owns 128 n and a batch slice; one atomic add per element at the end.
// Tensor path: WX = FK + Q + 1 <= 128 (WP = WX padded to 32 / 64 / 128) and N % 4 == 0 (the TMA row pitch of g_out / out).
// That holds the reference defaults (F = K = 8: WX = 101, N = 1024) for both methods.  Other shapes run the CUDA-core
// kernels below (chosen by shape only).
#include <stdlib.h>

#include "tc_ptx.cuh"

namespace ctr {
namespace pnn {
using namespace ctr::tc;

constexpr int NWG = 2;
constexpr int NTHREADS = (NWG + 1) * 128;
constexpr int TILE = NWG * WG_M;             // samples per CTA tile (forward, dx)
constexpr int FWD_NT = 64;                   // n per forward B tile (wgmma N)
constexpr int KB = 32;                       // tf32 per 128-byte swizzle row
constexpr int DW_BC = 32;                    // samples per dW chunk
constexpr int DW_NC = NWG * WG_M;            // n per dW CTA
constexpr int CHUNK_KS = 32;                 // k-steps per accumulation chain: 32 x 3 = 96 MMAs

__host__ __device__ inline int pair_index(int i, int j, int n) { return i * n - i * (i - 1) / 2 + (j - i); }   // i <= j
__host__ __device__ inline int64_t num_pairs(int64_t F, int64_t K, int method) {
  return method == 0 ? F * (F + 1) / 2 : K * (K + 1) / 2;
}
static inline int wpad(int64_t WX) { return WX <= 32 ? 32 : WX <= 64 ? 64 : 128; }
static inline int64_t pad_to(int64_t v, int64_t q) { return (v + q - 1) / q * q; }

__device__ __forceinline__ void consumers_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// (i, j) of upper-triangle pair q of an n x n matrix
__device__ __forceinline__ void pair_of(int q, int n, int& i, int& j) {
  i = 0;
  while (q >= n - i) { q -= n - i; ++i; }
  j = i + q;
}

// Wm[k, n]: k < FK linear_w; k < FK + Q the weight of pair feature k - FK (c factor included); k == WX - 1 bias (0 if null)
__device__ __forceinline__ float wm_value(const float* __restrict__ wlin, const float* __restrict__ wprod,
                                          const float* __restrict__ bias, int k, int n, int F, int K, int N, int method) {
  const int FK = F * K;
  if (k < FK) return __ldg(wlin + (size_t)k * N + n);
  const int q = k - FK;
  const int Q = method == 0 ? F * (F + 1) / 2 : K * (K + 1) / 2;
  if (q < Q) {
    int i, j;
    pair_of(q, method == 0 ? F : K, i, j);
    const float c = i == j ? 1.f : 2.f;
    if (method == 0) return c * __ldg(wprod + (size_t)n * F + i) * __ldg(wprod + (size_t)n * F + j);
    return c * __ldg(wprod + ((size_t)n * K + i) * K + j);
  }
  return bias != nullptr ? __ldg(bias + n) : 0.f;
}

// Writes Wm into dst as [rows][cols] (k_rows: rows are k, else rows are n), zero padded; split: hi | lo copies.
__global__ void pnn_prep_kernel(const float* __restrict__ wlin, const float* __restrict__ wprod, const float* __restrict__ bias,
                                float* __restrict__ dst, int F, int K, int N, int method, int WX, int rows, int cols,
                                int k_rows, int split) {
  const size_t total = (size_t)rows * cols;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(idx / cols), c = (int)(idx % cols);
    const int k = k_rows ? r : c, n = k_rows ? c : r;
    const float v = (k < WX && n < N) ? wm_value(wlin, wprod, bias, k, n, F, K, N, method) : 0.f;
    if (split) {
      const float hi = tf32_rna(v);
      dst[idx] = hi;
      dst[total + idx] = v - hi;
    } else {
      dst[idx] = v;
    }
  }
}

// dWm^T (N, WX) -> d_linear_w (FK, N), d_bias (N), d_inner_product_w (N, F) | d_outer_product_w (N, K, K)
__global__ void pnn_fold_kernel(const float* __restrict__ dwt, const float* __restrict__ wprod, float* __restrict__ d_wlin,
                                float* __restrict__ d_wprod, float* __restrict__ d_bias, int F, int K, int N, int method,
                                int WX) {
  const int FK = F * K;
  const size_t n_lin = (size_t)FK * N, n_prod = method == 0 ? (size_t)N * F : (size_t)N * K * K;
  const size_t total = n_lin + N + n_prod;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    if (idx < n_lin) {
      const int k = (int)(idx / N), n = (int)(idx % N);
      d_wlin[idx] = dwt[(size_t)n * WX + k];
    } else if (idx < n_lin + N) {
      const int n = (int)(idx - n_lin);
      d_bias[n] = dwt[(size_t)n * WX + WX - 1];
    } else {
      const size_t p = idx - n_lin - N;
      const float* dq = dwt + (size_t)(method == 0 ? p / F : p / (K * K)) * WX + FK;
      if (method == 0) {                      // d theta[n,f] = 2 sum_g dQ(min(f,g), max(f,g)) theta[n,g]
        const int n = (int)(p / F), f = (int)(p % F);
        float acc = 0.f;
        for (int g = 0; g < F; ++g)
          acc += dq[f <= g ? pair_index(f, g, F) : pair_index(g, f, F)] * __ldg(wprod + (size_t)n * F + g);
        d_wprod[p] = 2.f * acc;
      } else {                                // upper triangle c * dQ(k,l); the strictly lower triangle is never read
        const int kl = (int)(p % (K * K)), k = kl / K, l = kl % K;
        d_wprod[p] = k <= l ? (k == l ? 1.f : 2.f) * dq[pair_index(k, l, K)] : 0.f;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ feature generation
// Column descriptors of xt: {x >= 0, y < 0}: e_flat[x];  {x, y >= 0}: pair (x, y);  {-1, -1}: 1 (bias);  {-2, -1}: 0 (pad)
__device__ __forceinline__ int2 column_info(int col, int FK, int Q, int pn) {
  if (col < FK) return make_int2(col, -1);
  if (col < FK + Q) {
    int i, j;
    pair_of(col - FK, pn, i, j);
    return make_int2(i, j);
  }
  return make_int2(col == FK + Q ? -1 : -2, -1);
}
// xt[col] of one sample: er = its e row (FK floats), sr = its field sum s (K floats, OPNN only)
template <int METHOD>
__device__ __forceinline__ float feature(int2 ci, const float* er, const float* sr, int K) {
  if (ci.y < 0) return ci.x >= 0 ? er[ci.x] : (ci.x == -1 ? 1.f : 0.f);
  if (METHOD == 1) return sr[ci.x] * sr[ci.y];
  const float* a = er + ci.x * K;
  const float* b = er + ci.y * K;
  float acc = 0.f;
  for (int k = 0; k < K; ++k) acc = fmaf(a[k], b[k], acc);
  return acc;
}

// ================================================================================================= forward (wgmma)
__host__ __device__ inline int fwd_stage_bytes(int WP) { return 2 * (WP / KB) * FWD_NT * 128; }
__host__ __device__ inline int fwd_smem_bytes(int WP, int SB, int FK) {
  return SB * fwd_stage_bytes(WP) + NWG * WG_M * (FK + 1) * 4 + NWG * WG_M * 16 * 4 + WP * 8 + 16 * SB;
}

template <int WP, int SB, int METHOD>
__global__ void __launch_bounds__(NTHREADS, 1)
pnn_fwd_tc_kernel(const __grid_constant__ CUtensorMap tmap_w, const float* __restrict__ e, float* __restrict__ out, int B,
                  int F, int K, int N, int NP, int nsplit) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr int stage_bytes = 2 * (WP / KB) * FWD_NT * 128;
  constexpr int copy_bytes = stage_bytes / 2;
  const int FK = F * K, FKP = FK + 1;
  const int Q = METHOD == 0 ? F * (F + 1) / 2 : K * (K + 1) / 2;
  float* esm = reinterpret_cast<float*>(smem + SB * stage_bytes);          // [2][64][FK+1]
  float* ssm = esm + NWG * WG_M * FKP;                                       // [2][64][16]
  int2* cinfo = reinterpret_cast<int2*>(ssm + NWG * WG_M * 16);              // [WP]
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar0 = smem_u32(cinfo + WP);
  auto full_b = [&](int s) { return bar0 + 8 * s; };
  auto empty_b = [&](int s) { return bar0 + 8 * (SB + s); };

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_btiles = (B + TILE - 1) / TILE, NT = NP / FWD_NT;
  const int per_split = (NT + nsplit - 1) / nsplit;
  const int n_items = n_btiles * nsplit;

  for (int c = threadIdx.x; c < WP; c += blockDim.x) cinfo[c] = column_info(c, FK, Q, METHOD == 0 ? F : K);
  if (threadIdx.x == 0) {
    for (int s = 0; s < SB; ++s) { mbar_init(full_b(s), 1); mbar_init(empty_b(s), NWG * 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= NWG * 4) {
    // ============================ TMA producer: Wm^T tiles [64 n x WP] (hi, lo) ============================
    setmaxnreg_dec<40>();
    if (warp == NWG * 4 && lane == 0) {
      int s = 0, ph = 0;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int nt0 = (item % nsplit) * per_split, nt1 = min(NT, nt0 + per_split);
        for (int nt = nt0; nt < nt1; ++nt) {
          mbar_wait(empty_b(s), ph ^ 1);
          const uint32_t dst = sbase + s * stage_bytes;
          mbar_expect_tx(full_b(s), (uint32_t)stage_bytes);
          for (int kb = 0; kb < WP / KB; ++kb) {
            tma_load_2d(dst + kb * FWD_NT * 128, &tmap_w, kb * KB, nt * FWD_NT, full_b(s));
            tma_load_2d(dst + copy_bytes + kb * FWD_NT * 128, &tmap_w, kb * KB, NP + nt * FWD_NT, full_b(s));
          }
          if (++s == SB) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // ============================ consumers ============================
  setmaxnreg_inc<232>();
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3, tw = threadIdx.x & 127;
  float* er = esm + wg * WG_M * FKP;
  float* sr = ssm + wg * WG_M * 16;
  int s = 0, ph = 0;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int bt = item / nsplit;
    const int nt0 = (item % nsplit) * per_split, nt1 = min(NT, nt0 + per_split);
    const long long base = (long long)bt * TILE + wg * WG_M;
    // stage this warpgroup's 64 e rows (one contiguous block of e) and, for OPNN, their field sums
    for (int idx = tw; idx < WG_M * FK; idx += 128) {
      const int row = idx / FK, c = idx % FK;
      er[row * FKP + c] = base + row < B ? __ldg(e + (size_t)base * FK + idx) : 0.f;
    }
    wg_bar_sync(1 + wg);
    if (METHOD == 1) {
      for (int idx = tw; idx < WG_M * K; idx += 128) {
        const int row = idx / K, l = idx % K;
        float acc = 0.f;
        for (int f = 0; f < F; ++f) acc += er[row * FKP + f * K + l];
        sr[row * 16 + l] = acc;
      }
      wg_bar_sync(1 + wg);
    }
    // A fragments of xt: a[q] = xt[16w + g + 8(q&1)][8ks + t + 4(q>>1)]
    uint32_t ah[WP / 8][4], al[WP / 8][4];
    const int r0 = w * 16 + g;
#pragma unroll
    for (int ks = 0; ks < WP / 8; ++ks) {
      float a[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int row = r0 + 8 * (q & 1), col = 8 * ks + t + 4 * (q >> 1);
        a[q] = feature<METHOD>(cinfo[col], er + row * FKP, sr + row * 16, K);
      }
      tf32_split(a, ah[ks], al[ks]);
    }
    wg_bar_sync(1 + wg);                      // the e rows may be restaged once every thread has its fragments
    const bool v0 = base + r0 < B, v1 = base + r0 + 8 < B;
    float* o0 = out + (size_t)(base + r0) * N;
    float* o1 = o0 + (size_t)8 * N;
    for (int nt = nt0; nt < nt1; ++nt) {
      float d[FWD_NT / 2];
      mbar_wait(full_b(s), ph);
      const uint64_t bhi = gmma_desc_kmajor(sbase + s * stage_bytes, 128);
      const uint64_t blo = gmma_desc_kmajor(sbase + s * stage_bytes + copy_bytes, 128);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < WP / 8; ++ks) {
        const uint64_t off = (uint64_t)((ks >> 2) * (FWD_NT * 128 / 16) + 2 * (ks & 3));
        wgmma_tf32_rs<FWD_NT>(d, al[ks], bhi + off, ks > 0 ? 1 : 0);     // small terms first
        wgmma_tf32_rs<FWD_NT>(d, ah[ks], blo + off, 1);
        wgmma_tf32_rs<FWD_NT>(d, ah[ks], bhi + off, 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int ks = 0; ks < WP / 8; ++ks) { wgmma_keep(ah[ks]); wgmma_keep(al[ks]); }
      if (lane == 0) mbar_arrive(empty_b(s));
      if (++s == SB) { s = 0; ph ^= 1; }
#pragma unroll
      for (int c = 0; c < FWD_NT / 8; ++c) {
#pragma unroll
        for (int x = 0; x < 2; ++x) {
          const int n = nt * FWD_NT + 8 * c + 2 * t + x;
          if (n < N) {
            if (v0) o0[n] = fmaxf(d[4 * c + x], 0.f);
            if (v1) o1[n] = fmaxf(d[4 * c + 2 + x], 0.f);
          }
        }
      }
    }
  }
}

// ================================================================================================= backward dx (wgmma)
__host__ __device__ inline int dx_smem_bytes(int WP, int SB) {
  return SB * 2 * WP * 128 + NWG * WG_M * (WP + 1) * 4 + NWG * WG_M * 16 * 4 + 16 * SB;
}

template <int WP, int SB, int METHOD>
__global__ void __launch_bounds__(NTHREADS, 1)
pnn_bwd_dx_tc_kernel(const __grid_constant__ CUtensorMap tmap_w, const float* __restrict__ e, const float* __restrict__ outv,
                     const float* __restrict__ g_out, float* __restrict__ d_e, int B, int F, int K, int N, int NPK) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr int copy_bytes = WP * 128;
  constexpr int stage_bytes = 2 * copy_bytes;
  constexpr int LD = WP + 1;
  const int FK = F * K;
  float* dsm = reinterpret_cast<float*>(smem + SB * stage_bytes);          // [2][64][WP+1]  dxt of the tile
  float* ssm = dsm + NWG * WG_M * LD;                                        // [2][64][16]    s (OPNN)
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar0 = smem_u32(ssm + NWG * WG_M * 16);
  auto full_b = [&](int s) { return bar0 + 8 * s; };
  auto empty_b = [&](int s) { return bar0 + 8 * (SB + s); };

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_tiles = (B + TILE - 1) / TILE, nkb = NPK / KB;

  if (threadIdx.x == 0) {
    for (int s = 0; s < SB; ++s) { mbar_init(full_b(s), 1); mbar_init(empty_b(s), NWG * 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= NWG * 4) {
    // ============================ TMA producer: Wm tiles [WP k x 32 n] (hi, lo) ============================
    setmaxnreg_dec<40>();
    if (warp == NWG * 4 && lane == 0) {
      int s = 0, ph = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(empty_b(s), ph ^ 1);
          const uint32_t dst = sbase + s * stage_bytes;
          mbar_expect_tx(full_b(s), (uint32_t)stage_bytes);
          tma_load_2d(dst, &tmap_w, kb * KB, 0, full_b(s));
          tma_load_2d(dst + copy_bytes, &tmap_w, kb * KB, WP, full_b(s));
          if (++s == SB) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // ============================ consumers: G fragments per 32-column block, dxt, chain rule ============================
  setmaxnreg_inc<232>();
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3, tw = threadIdx.x & 127;
  float* ds = dsm + wg * WG_M * LD;
  float* sr = ssm + wg * WG_M * 16;
  int s = 0, ph = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long base = (long long)tile * TILE + wg * WG_M;
    const int r0 = w * 16 + g;
    const bool valid[2] = {base + r0 < B, base + r0 + 8 < B};
    const float* gp[2] = {g_out + (size_t)(base + r0) * N, g_out + (size_t)(base + r0 + 8) * N};
    const float* op[2] = {outv + (size_t)(base + r0) * N, outv + (size_t)(base + r0 + 8) * N};
    float acc[WP / 2], dacc[WP / 2];
#pragma unroll
    for (int q = 0; q < WP / 2; ++q) { acc[q] = 0.f; dacc[q] = 0.f; }
    for (int kb = 0; kb < nkb; ++kb) {
      uint32_t gh[4][4], gl[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        float a[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int rr = q & 1, n = kb * KB + 8 * ks + t + 4 * (q >> 1);
          a[q] = (valid[rr] && n < N && __ldg(op[rr] + n) > 0.f) ? __ldg(gp[rr] + n) : 0.f;
        }
        tf32_split(a, gh[ks], gl[ks]);
      }
      const bool chain_start = (kb * 4) % CHUNK_KS == 0;
      mbar_wait(full_b(s), ph);
      const uint64_t bhi = gmma_desc_kmajor(sbase + s * stage_bytes, 128);
      const uint64_t blo = gmma_desc_kmajor(sbase + s * stage_bytes + copy_bytes, 128);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        wgmma_tf32_rs<WP>(dacc, gl[ks], bhi + 2 * ks, (chain_start && ks == 0) ? 0 : 1);
        wgmma_tf32_rs<WP>(dacc, gh[ks], blo + 2 * ks, 1);
        wgmma_tf32_rs<WP>(dacc, gh[ks], bhi + 2 * ks, 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) { wgmma_keep(gh[ks]); wgmma_keep(gl[ks]); }
      if (lane == 0) mbar_arrive(empty_b(s));
      if (++s == SB) { s = 0; ph ^= 1; }
      if (((kb + 1) * 4) % CHUNK_KS == 0 || kb + 1 == nkb) {
#pragma unroll
        for (int q = 0; q < WP / 2; ++q) acc[q] += dacc[q];
      }
    }
    // ---------------- epilogue: dxt fragment -> ds[row][col]; d_e = dxt_lin + chain rule through the pair features
#pragma unroll
    for (int c = 0; c < WP / 8; ++c) {
#pragma unroll
      for (int x = 0; x < 2; ++x) {
        ds[r0 * LD + 8 * c + 2 * t + x] = acc[4 * c + x];
        ds[(r0 + 8) * LD + 8 * c + 2 * t + x] = acc[4 * c + 2 + x];
      }
    }
    if (METHOD == 1) {
      for (int idx = tw; idx < WG_M * K; idx += 128) {
        const int row = idx / K, l = idx % K;
        float v = 0.f;
        if (base + row < B)
          for (int f = 0; f < F; ++f) v += __ldg(e + (size_t)(base + row) * FK + f * K + l);
        sr[row * 16 + l] = v;
      }
    }
    wg_bar_sync(1 + wg);
    for (int idx = tw; idx < WG_M * FK; idx += 128) {
      const int row = idx / FK, fk = idx % FK;
      if (base + row >= B) break;
      const float* dq = ds + row * LD + FK;
      float v = ds[row * LD + fk];
      const int f = fk / K, k = fk % K;
      if (METHOD == 0) {             // d e_f += sum_g dq(f,g) (1 + [f == g]) e_g
        const float* eb = e + (size_t)(base + row) * FK + k;
        for (int g2 = 0; g2 < F; ++g2) {
          const float dqv = dq[f <= g2 ? pair_index(f, g2, F) : pair_index(g2, f, F)];
          v += (g2 == f ? 2.f : 1.f) * dqv * __ldg(eb + g2 * K);
        }
      } else {                       // d e_f += ds_k = sum_l dq(k,l) (1 + [k == l]) s_l
        for (int l = 0; l < K; ++l) {
          const float dqv = dq[k <= l ? pair_index(k, l, K) : pair_index(l, k, K)];
          v += (l == k ? 2.f : 1.f) * dqv * sr[row * 16 + l];
        }
      }
      d_e[(size_t)base * FK + idx] = v;
    }
    wg_bar_sync(1 + wg);
  }
}

// ================================================================================================= backward dW (wgmma)
__host__ __device__ inline int dw_smem_bytes(int WP, int SB, int FK, int K) {
  return SB * (2 * WP * 128 + 2 * DW_BC * DW_NC * 4) + DW_BC * (FK + 1) * 4 + DW_BC * (K + 1) * 4 + WP * 8 + 16 * SB;
}

template <int WP, int METHOD>
__global__ void __launch_bounds__(NTHREADS, 1)
pnn_bwd_dw_tc_kernel(const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ CUtensorMap tmap_o,
                     const float* __restrict__ e, float* __restrict__ dwt, int B, int F, int K, int N, int WX, int ngroups,
                     int nslices, int SB) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr int xt_bytes = 2 * WP * 128;                      // xt^T tiles [WP k x 32 samples] (hi | lo), 128B-swizzled
  constexpr int go_bytes = DW_BC * DW_NC * 4;                 // one g_out or out chunk [32 samples x 128 n]
  const int FK = F * K, FKP = FK + 1;
  const int Q = METHOD == 0 ? F * (F + 1) / 2 : K * (K + 1) / 2;
  uint8_t* xts = smem;                                        // SB tiles (1024-byte aligned)
  float* gos = reinterpret_cast<float*>(smem + SB * xt_bytes);            // SB x (g | out)
  float* esm = gos + SB * 2 * DW_BC * DW_NC;                               // [32][FK+1]
  float* ssm = esm + DW_BC * FKP;                                          // [32][K+1]
  int2* cinfo = reinterpret_cast<int2*>(ssm + DW_BC * (K + 1));            // [WP]
  const uint32_t bar0 = smem_u32(cinfo + WP);
  auto full_b = [&](int s) { return bar0 + 8 * s; };
  auto empty_b = [&](int s) { return bar0 + 8 * (SB + s); };

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int group = blockIdx.x % ngroups, slice = blockIdx.x / ngroups;
  const int n_chunks = (B + DW_BC - 1) / DW_BC;
  const int per_slice = (n_chunks + nslices - 1) / nslices;
  const int c_beg = min(n_chunks, slice * per_slice), c_end = min(n_chunks, c_beg + per_slice);
  const int n0 = group * DW_NC;

  for (int c = threadIdx.x; c < WP; c += blockDim.x) cinfo[c] = column_info(c, FK, Q, METHOD == 0 ? F : K);
  if (threadIdx.x == 0) {
    for (int s = 0; s < SB; ++s) { mbar_init(full_b(s), 1); mbar_init(empty_b(s), NWG * 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= NWG * 4) {
    // ============================ TMA producer: g_out / out chunks [32 samples x 128 n] ============================
    setmaxnreg_dec<40>();
    if (warp == NWG * 4 && lane == 0) {
      int s = 0, ph = 0;
      for (int c = c_beg; c < c_end; ++c) {
        mbar_wait(empty_b(s), ph ^ 1);
        const uint32_t dst = smem_u32(gos + (size_t)s * 2 * DW_BC * DW_NC);
        mbar_expect_tx(full_b(s), (uint32_t)(2 * go_bytes));
        tma_load_2d(dst, &tmap_g, n0, c * DW_BC, full_b(s));
        tma_load_2d(dst + go_bytes, &tmap_o, n0, c * DW_BC, full_b(s));
        if (++s == SB) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ============================ consumers ============================
  setmaxnreg_inc<232>();
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3, ct = threadIdx.x;   // ct: 0..255
  float acc[WP / 2], dacc[WP / 2];
#pragma unroll
  for (int q = 0; q < WP / 2; ++q) { acc[q] = 0.f; dacc[q] = 0.f; }
  int s = 0, ph = 0;
  const int nl0 = wg * WG_M + w * 16 + g;                     // this thread's A rows: n0 + nl0 (+8)
  for (int c = c_beg; c < c_end; ++c) {
    const int b0 = c * DW_BC;
    // 1. stage the chunk's e rows (+ field sums) -- all 256 consumer threads
    for (int idx = ct; idx < DW_BC * FK; idx += 256) {
      const int row = idx / FK, col = idx % FK;
      esm[row * FKP + col] = b0 + row < B ? __ldg(e + (size_t)b0 * FK + idx) : 0.f;
    }
    consumers_bar();
    if (METHOD == 1) {
      for (int idx = ct; idx < DW_BC * K; idx += 256) {
        const int row = idx / K, l = idx % K;
        float v = 0.f;
        for (int f = 0; f < F; ++f) v += esm[row * FKP + f * K + l];
        ssm[row * (K + 1) + l] = v;
      }
      consumers_bar();
    }
    mbar_wait(full_b(s), ph);
    // 2. xt^T (tf32 hi | lo) into the stage's swizzled B tiles: element (k, b) at byte k*128 + 4b, 16-byte chunk XOR (k & 7)
    uint8_t* xt = xts + s * xt_bytes;
    for (int idx = ct; idx < WP * DW_BC; idx += 256) {
      const int k = idx / DW_BC, b = idx % DW_BC;
      const float v = b0 + b < B ? feature<METHOD>(cinfo[k], esm + b * FKP, ssm + b * (K + 1), K) : 0.f;
      const float hi = tf32_rna(v);
      const uint32_t o = (uint32_t)(k * 128 + b * 4);
      const uint32_t so = o ^ (((o >> 7) & 7u) << 4);
      *reinterpret_cast<float*>(xt + so) = hi;
      *reinterpret_cast<float*>(xt + WP * 128 + so) = v - hi;
    }
    fence_proxy_async();                                      // generic-proxy writes -> visible to wgmma
    consumers_bar();
    // 3. A fragments of G^T: a[q] = G[b = 8ks + t + 4(q>>1)][n = nl0 + 8(q&1)]
    const float* gs = gos + (size_t)s * 2 * DW_BC * DW_NC;
    const float* os = gs + DW_BC * DW_NC;
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      float a[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int b = 8 * ks + t + 4 * (q >> 1), nl = nl0 + 8 * (q & 1);
        a[q] = os[b * DW_NC + nl] > 0.f ? gs[b * DW_NC + nl] : 0.f;
      }
      tf32_split(a, ah[ks], al[ks]);
    }
    const bool chain_start = ((c - c_beg) * 4) % CHUNK_KS == 0;
    const uint64_t bhi = gmma_desc_kmajor(smem_u32(xt), 128);
    const uint64_t blo = gmma_desc_kmajor(smem_u32(xt + WP * 128), 128);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      wgmma_tf32_rs<WP>(dacc, al[ks], bhi + 2 * ks, (chain_start && ks == 0) ? 0 : 1);
      wgmma_tf32_rs<WP>(dacc, ah[ks], blo + 2 * ks, 1);
      wgmma_tf32_rs<WP>(dacc, ah[ks], bhi + 2 * ks, 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) { wgmma_keep(ah[ks]); wgmma_keep(al[ks]); }
    if (lane == 0) mbar_arrive(empty_b(s));
    if (++s == SB) { s = 0; ph ^= 1; }
    if (((c - c_beg + 1) * 4) % CHUNK_KS == 0 || c + 1 == c_end) {
#pragma unroll
      for (int q = 0; q < WP / 2; ++q) acc[q] += dacc[q];
    }
  }
  if (c_end > c_beg) {
#pragma unroll
    for (int cc = 0; cc < WP / 8; ++cc) {
#pragma unroll
      for (int x = 0; x < 2; ++x) {
        const int k = 8 * cc + 2 * t + x;
        if (k < WX) {
          if (n0 + nl0 < N) atomicAdd(dwt + (size_t)(n0 + nl0) * WX + k, acc[4 * cc + x]);
          if (n0 + nl0 + 8 < N) atomicAdd(dwt + (size_t)(n0 + nl0 + 8) * WX + k, acc[4 * cc + 2 + x]);
        }
      }
    }
  }
}

// ================================================================================================= CUDA-core path
constexpr int SIMPLE_SPB = 4;                 // samples per forward CTA iteration

template <int METHOD>
__device__ void features_to_smem(const float* __restrict__ erow_g, float* xs, float* es, float* ss, int F, int K, int WX) {
  const int FK = F * K;
  for (int i = threadIdx.x; i < FK; i += blockDim.x) es[i] = __ldg(erow_g + i);
  __syncthreads();
  if (METHOD == 1) {
    for (int l = threadIdx.x; l < K; l += blockDim.x) {
      float v = 0.f;
      for (int f = 0; f < F; ++f) v += es[f * K + l];
      ss[l] = v;
    }
    __syncthreads();
  }
  const int Q = METHOD == 0 ? F * (F + 1) / 2 : K * (K + 1) / 2;
  for (int k = threadIdx.x; k < WX; k += blockDim.x) xs[k] = feature<METHOD>(column_info(k, FK, Q, METHOD == 0 ? F : K), es, ss, K);
}

// out[b, n] = relu(sum_k xt[b,k] Wm[k,n]); Wm as [WX][N]
template <int METHOD>
__global__ void __launch_bounds__(256)
pnn_fwd_simple_kernel(const float* __restrict__ e, const float* __restrict__ wm, float* __restrict__ out, int B, int F, int K,
                      int N, int WX) {
  extern __shared__ __align__(16) float sm[];
  const int FK = F * K;
  float* xs = sm;                               // [SPB][WX]
  float* es = xs + SIMPLE_SPB * WX;             // [FK]
  float* ss = es + FK;                          // [K]
  for (int b0 = blockIdx.x * SIMPLE_SPB; b0 < B; b0 += gridDim.x * SIMPLE_SPB) {
    for (int j = 0; j < SIMPLE_SPB; ++j) {
      __syncthreads();
      if (b0 + j < B) features_to_smem<METHOD>(e + (size_t)(b0 + j) * FK, xs + j * WX, es, ss, F, K, WX);
    }
    __syncthreads();
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      float acc[SIMPLE_SPB] = {};
      for (int k = 0; k < WX; ++k) {
        const float wv = __ldg(wm + (size_t)k * N + n);
#pragma unroll
        for (int j = 0; j < SIMPLE_SPB; ++j) acc[j] = fmaf(xs[j * WX + k], wv, acc[j]);
      }
#pragma unroll
      for (int j = 0; j < SIMPLE_SPB; ++j)
        if (b0 + j < B) out[(size_t)(b0 + j) * N + n] = fmaxf(acc[j], 0.f);
    }
  }
}

// d_e of one sample per CTA iteration; Wm as [N][WX]
template <int METHOD>
__global__ void __launch_bounds__(256)
pnn_bwd_dx_simple_kernel(const float* __restrict__ e, const float* __restrict__ wmt, const float* __restrict__ outv,
                         const float* __restrict__ g_out, float* __restrict__ d_e, int B, int F, int K, int N, int WX) {
  extern __shared__ __align__(16) float sm[];
  const int FK = F * K;
  float* gs = sm;                 // [N]
  float* es = gs + N;             // [FK]
  float* ss = es + FK;            // [K]
  float* dx = ss + K;             // [WX]
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
      const size_t o = (size_t)b * N + n;
      gs[n] = __ldg(outv + o) > 0.f ? __ldg(g_out + o) : 0.f;
    }
    for (int i = threadIdx.x; i < FK; i += blockDim.x) es[i] = __ldg(e + (size_t)b * FK + i);
    __syncthreads();
    if (METHOD == 1)
      for (int l = threadIdx.x; l < K; l += blockDim.x) {
        float v = 0.f;
        for (int f = 0; f < F; ++f) v += es[f * K + l];
        ss[l] = v;
      }
    for (int k = threadIdx.x; k < WX; k += blockDim.x) {
      float acc = 0.f;
      for (int n = 0; n < N; ++n) acc = fmaf(gs[n], __ldg(wmt + (size_t)n * WX + k), acc);
      dx[k] = acc;
    }
    __syncthreads();
    const float* dq = dx + FK;
    for (int fk = threadIdx.x; fk < FK; fk += blockDim.x) {
      const int f = fk / K, k = fk % K;
      float v = dx[fk];
      if (METHOD == 0) {
        for (int g2 = 0; g2 < F; ++g2)
          v += (g2 == f ? 2.f : 1.f) * dq[f <= g2 ? pair_index(f, g2, F) : pair_index(g2, f, F)] * es[g2 * K + k];
      } else {
        for (int l = 0; l < K; ++l)
          v += (l == k ? 2.f : 1.f) * dq[k <= l ? pair_index(k, l, K) : pair_index(l, k, K)] * ss[l];
      }
      d_e[(size_t)b * FK + fk] = v;
    }
  }
}

// dWm^T[n, k] += sum_b G[b,n] xt[b,k]: grid (ceil(WX / PC), ceil(N / 256), slices); one atomic add per element per CTA
constexpr int SIMPLE_PC = 16;
template <int METHOD>
__global__ void __launch_bounds__(256)
pnn_bwd_dw_simple_kernel(const float* __restrict__ e, const float* __restrict__ outv, const float* __restrict__ g_out,
                         float* __restrict__ dwt, int B, int F, int K, int N, int WX) {
  extern __shared__ __align__(16) float sm[];
  const int FK = F * K;
  const int Q = METHOD == 0 ? F * (F + 1) / 2 : K * (K + 1) / 2;
  float* es = sm;                 // [FK]
  float* ss = es + FK;            // [K]
  float* zs = ss + K;             // [PC]
  const int k0 = blockIdx.x * SIMPLE_PC, n = blockIdx.y * blockDim.x + threadIdx.x;
  float acc[SIMPLE_PC] = {};
  for (int b = blockIdx.z; b < B; b += gridDim.z) {
    __syncthreads();
    for (int i = threadIdx.x; i < FK; i += blockDim.x) es[i] = __ldg(e + (size_t)b * FK + i);
    __syncthreads();
    if (METHOD == 1) {
      for (int l = threadIdx.x; l < K; l += blockDim.x) {
        float v = 0.f;
        for (int f = 0; f < F; ++f) v += es[f * K + l];
        ss[l] = v;
      }
      __syncthreads();
    }
    for (int q = threadIdx.x; q < SIMPLE_PC; q += blockDim.x)
      zs[q] = k0 + q < WX ? feature<METHOD>(column_info(k0 + q, FK, Q, METHOD == 0 ? F : K), es, ss, K) : 0.f;
    __syncthreads();
    if (n < N) {
      const size_t o = (size_t)b * N + n;
      const float gv = __ldg(outv + o) > 0.f ? __ldg(g_out + o) : 0.f;
#pragma unroll
      for (int q = 0; q < SIMPLE_PC; ++q) acc[q] = fmaf(zs[q], gv, acc[q]);
    }
  }
  if (n < N)
#pragma unroll
    for (int q = 0; q < SIMPLE_PC; ++q)
      if (k0 + q < WX) atomicAdd(dwt + (size_t)n * WX + k0 + q, acc[q]);
}

}  // namespace pnn
}  // namespace ctr

// ------------------------------------------------------------------------------------------------ host
using namespace ctr;
using namespace ctr::pnn;

namespace {

struct PnnShape {
  int64_t F, K, N, FK, Q, WX;
  int method;
  bool tc;                         // tensor path
  int WP;                          // WX padded for wgmma (tensor path)
  int64_t NP, NPK;                 // N padded to 64 (forward tiles) / 32 (backward K-blocks)
  int64_t w_floats, d_offset;      // workspace: derived weights | dWm^T (N, WX) at byte offset d_offset
};

PnnShape shape_of(int64_t F, int64_t K, int64_t N, int method) {
  PnnShape s;
  s.F = F; s.K = K; s.N = N; s.method = method;
  s.FK = F * K;
  s.Q = num_pairs(F, K, method);
  s.WX = s.FK + s.Q + 1;
  s.tc = s.WX <= 128 && N % 4 == 0;
  s.WP = wpad(s.WX);
  s.NP = pad_to(N, FWD_NT);
  s.NPK = pad_to(N, KB);
  s.w_floats = s.tc ? 2 * s.WP * (s.NP > s.NPK ? s.NP : s.NPK) : s.WX * N;
  s.d_offset = pad_to(s.w_floats * (int64_t)sizeof(float), 128);
  return s;
}

int64_t workspace_of(const PnnShape& s) { return s.d_offset + pad_to(s.N * s.WX * (int64_t)sizeof(float), 128); }

int check_pnn(const char* fn, int64_t B, int64_t F, int64_t K, int64_t N, int method) {
  CTR_REQUIRE(B >= 0 && F >= 1 && K >= 1 && N >= 1, "%s: bad sizes B=%lld F=%lld K=%lld N=%lld", fn, (long long)B,
              (long long)F, (long long)K, (long long)N);
  CTR_REQUIRE(method == 0 || method == 1, "%s: method must be 0 (IPNN) or 1 (OPNN), got %d", fn, method);
  CTR_UNSUPPORTED(F > 4096 || K > 4096 || F * K > 65536 || N > (1 << 20) || B > 0x7fffff00LL,
                  "%s: problem too large (F=%lld K=%lld N=%lld B=%lld)", fn, (long long)F, (long long)K, (long long)N,
                  (long long)B);
  CTR_UNSUPPORTED(num_pairs(F, K, method) * N > (1LL << 31), "%s: product weights too large", fn);
  return CTR_OK;
}

int check_workspace(const char* fn, const PnnShape& s, void* workspace, int64_t workspace_bytes) {
  const int64_t need = workspace_of(s);
  CTR_REQUIRE(workspace != nullptr && workspace_bytes >= need,
              "%s: workspace of %lld bytes required (ctr_pnn_workspace_bytes), got %lld", fn, (long long)need,
              (long long)workspace_bytes);
  CTR_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 127) == 0, "%s: workspace must be 128-byte aligned", fn);
  return CTR_OK;
}

int grid_for(size_t total, int cap) { return (int)((total + 255) / 256 < (size_t)cap ? (total + 255) / 256 : (size_t)cap); }

int encode_2d(const char* fn, CUtensorMap* map, const void* base, uint64_t inner, uint64_t outer, uint32_t box_inner,
              uint32_t box_outer, CUtensorMapSwizzle sw) {
  EncodeTiledFn enc = encode_tiled();
  if (enc == nullptr) {
    set_error("%s: cuTensorMapEncodeTiled is not available from the driver", fn);
    return CTR_ERR_CUDA;
  }
  const cuuint64_t gdim[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  const cuuint64_t gstr[1] = {(cuuint64_t)inner * sizeof(float)};
  const cuuint32_t box[2] = {box_inner, box_outer};
  const cuuint32_t es[2] = {1, 1};
  CUresult cr = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), gdim, gstr, box, es,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    set_error("%s: cuTensorMapEncodeTiled failed with CUresult %d", fn, (int)cr);
    return CTR_ERR_CUDA;
  }
  return CTR_OK;
}

int set_smem(const void* k, size_t bytes) {
  if (bytes > 48 * 1024) CTR_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return CTR_OK;
}

constexpr size_t SMEM_CAP = 226 * 1024;     // dynamic shared memory per CTA on sm_90 (227 KB) less slack

}  // namespace

extern "C" int ctr_pnn_workspace_bytes(int64_t F, int64_t K, int64_t N, int method, int64_t* bytes) {
  int rc = check_pnn("ctr_pnn_workspace_bytes", 0, F, K, N, method);
  if (rc) return rc;
  CTR_REQUIRE(bytes != nullptr, "ctr_pnn_workspace_bytes: null argument");
  *bytes = workspace_of(shape_of(F, K, N, method));
  return CTR_OK;
}

extern "C" int ctr_pnn_fwd(const float* e, const float* wlin, const float* wprod, const float* bias, int64_t B, int64_t F,
                           int64_t K, int64_t N, int method, float* out, void* workspace, int64_t workspace_bytes,
                           void* stream) {
  static const char* fn = "ctr_pnn_fwd";
  int rc = check_pnn(fn, B, F, K, N, method);
  if (rc) return rc;
  CTR_REQUIRE(e && wlin && wprod && bias && out, "ctr_pnn_fwd: null argument");
  const PnnShape s = shape_of(F, K, N, method);
  rc = check_workspace(fn, s, workspace, workspace_bytes);
  if (rc) return rc;
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  float* ws = static_cast<float*>(workspace);
  const int sms = sm_count();
  if (s.tc) {
    const size_t total = (size_t)s.NP * s.WP;
    pnn_prep_kernel<<<grid_for(total, 2048), 256, 0, st>>>(wlin, wprod, bias, ws, (int)F, (int)K, (int)N, method, (int)s.WX,
                                                         (int)s.NP, s.WP, 0, 1);
    CTR_CHECK_LAUNCH("ctr_pnn_fwd(prep)");
    CUtensorMap tmap;
    rc = encode_2d(fn, &tmap, ws, s.WP, 2 * s.NP, KB, FWD_NT, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
    const int n_btiles = (int)((B + TILE - 1) / TILE), NT = (int)(s.NP / FWD_NT);
    int nsplit = sms / n_btiles;                  // small batches: split the N loop across CTAs as well
    if (nsplit < 1) nsplit = 1;
    if (nsplit > NT) nsplit = NT;
    const long long items = (long long)n_btiles * nsplit;
    const int grid = (int)(items < sms ? items : sms);
#define PNN_FWD(WP_, SB_, M_)                                                                                            \
  {                                                                                                                      \
    const size_t smem = fwd_smem_bytes(WP_, SB_, (int)s.FK) + 1024;                                                      \
    auto k = pnn_fwd_tc_kernel<WP_, SB_, M_>;                                                                            \
    CTR_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                           \
    k<<<grid, NTHREADS, smem, st>>>(tmap, e, out, (int)B, (int)F, (int)K, (int)N, (int)s.NP, nsplit);                    \
  }
    if (method == 0) {
      if (s.WP == 32) PNN_FWD(32, 4, 0) else if (s.WP == 64) PNN_FWD(64, 3, 0) else PNN_FWD(128, 2, 0)
    } else {
      if (s.WP == 32) PNN_FWD(32, 4, 1) else if (s.WP == 64) PNN_FWD(64, 3, 1) else PNN_FWD(128, 2, 1)
    }
#undef PNN_FWD
    CTR_CHECK_LAUNCH("ctr_pnn_fwd(wgmma)");
    return CTR_OK;
  }
  const size_t smem = sizeof(float) * (size_t)(SIMPLE_SPB * s.WX + s.FK + s.K);
  CTR_UNSUPPORTED(smem > SMEM_CAP, "ctr_pnn_fwd: F*K=%lld too large for the CUDA-core path", (long long)s.FK);
  pnn_prep_kernel<<<grid_for((size_t)s.WX * N, 4096), 256, 0, st>>>(wlin, wprod, bias, ws, (int)F, (int)K, (int)N, method,
                                                                   (int)s.WX, (int)s.WX, (int)N, 1, 0);
  CTR_CHECK_LAUNCH("ctr_pnn_fwd(prep)");
  const int64_t groups = (B + SIMPLE_SPB - 1) / SIMPLE_SPB;
  const int grid = (int)(groups < (int64_t)sms * 4 ? groups : (int64_t)sms * 4);
  if (method == 0) {
    rc = set_smem((const void*)pnn_fwd_simple_kernel<0>, smem);
    if (rc) return rc;
    pnn_fwd_simple_kernel<0><<<grid, 256, smem, st>>>(e, ws, out, (int)B, (int)F, (int)K, (int)N, (int)s.WX);
  } else {
    rc = set_smem((const void*)pnn_fwd_simple_kernel<1>, smem);
    if (rc) return rc;
    pnn_fwd_simple_kernel<1><<<grid, 256, smem, st>>>(e, ws, out, (int)B, (int)F, (int)K, (int)N, (int)s.WX);
  }
  CTR_CHECK_LAUNCH("ctr_pnn_fwd(simple)");
  return CTR_OK;
}

extern "C" int ctr_pnn_bwd(const float* e, const float* wlin, const float* wprod, const float* out, const float* g_out,
                           int64_t B, int64_t F, int64_t K, int64_t N, int method, float* d_e, float* d_wlin,
                           float* d_wprod, float* d_bias, void* workspace, int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_pnn_bwd";
  int rc = check_pnn(fn, B, F, K, N, method);
  if (rc) return rc;
  CTR_REQUIRE(e && wlin && wprod && out && g_out && d_e && d_wlin && d_wprod && d_bias, "ctr_pnn_bwd: null argument");
  const PnnShape s = shape_of(F, K, N, method);
  rc = check_workspace(fn, s, workspace, workspace_bytes);
  if (rc) return rc;
  cudaStream_t st = as_stream(stream);
  float* ws = static_cast<float*>(workspace);
  float* dwt = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + s.d_offset);
  const int sms = sm_count();
  CTR_CUDA(cudaMemsetAsync(dwt, 0, sizeof(float) * (size_t)N * s.WX, st));
  if (B > 0 && s.tc) {
    CTR_REQUIRE(aligned16(out) && aligned16(g_out), "ctr_pnn_bwd: out and g_out must be 16-byte aligned");
    const size_t total = (size_t)s.WP * s.NPK;
    pnn_prep_kernel<<<grid_for(total, 2048), 256, 0, st>>>(wlin, wprod, nullptr, ws, (int)F, (int)K, (int)N, method,
                                                         (int)s.WX, s.WP, (int)s.NPK, 1, 1);
    CTR_CHECK_LAUNCH("ctr_pnn_bwd(prep)");
    // ---- d_e: Wm (hi | lo) as [2 WP rows x NPK], one [WP x 32] swizzled box per K-block
    {
      CUtensorMap tmap;
      rc = encode_2d(fn, &tmap, ws, s.NPK, 2 * s.WP, KB, s.WP, CU_TENSOR_MAP_SWIZZLE_128B);
      if (rc) return rc;
      const int tiles = (int)((B + TILE - 1) / TILE);
      const int grid = tiles < sms ? tiles : sms;
#define PNN_DX(WP_, M_)                                                                                                \
  {                                                                                                                    \
    const size_t smem = dx_smem_bytes(WP_, 4) + 1024;                                                                  \
    auto k = pnn_bwd_dx_tc_kernel<WP_, 4, M_>;                                                                         \
    CTR_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                         \
    k<<<grid, NTHREADS, smem, st>>>(tmap, e, out, g_out, d_e, (int)B, (int)F, (int)K, (int)N, (int)s.NPK);             \
  }
      if (method == 0) {
        if (s.WP == 32) PNN_DX(32, 0) else if (s.WP == 64) PNN_DX(64, 0) else PNN_DX(128, 0)
      } else {
        if (s.WP == 32) PNN_DX(32, 1) else if (s.WP == 64) PNN_DX(64, 1) else PNN_DX(128, 1)
      }
#undef PNN_DX
      CTR_CHECK_LAUNCH("ctr_pnn_bwd(dx, wgmma)");
    }
    // ---- dWm^T: g_out and out as [B rows x N], boxes of [32 samples x 128 n] (out-of-range rows / columns arrive as zeros)
    {
      CUtensorMap tg, to;
      rc = encode_2d(fn, &tg, g_out, N, B, DW_NC, DW_BC, CU_TENSOR_MAP_SWIZZLE_NONE);
      if (rc) return rc;
      rc = encode_2d(fn, &to, out, N, B, DW_NC, DW_BC, CU_TENSOR_MAP_SWIZZLE_NONE);
      if (rc) return rc;
      const int ngroups = (int)((N + DW_NC - 1) / DW_NC);
      const int64_t chunks = (B + DW_BC - 1) / DW_BC;
      int nslices = sms / ngroups;
      if (nslices < 1) nslices = 1;
      if (nslices > chunks) nslices = (int)chunks;
      const int grid = ngroups * nslices;
      const size_t fixed = dw_smem_bytes(s.WP, 0, (int)s.FK, (int)s.K) + 1024;
      const size_t stage = (size_t)dw_smem_bytes(s.WP, 1, (int)s.FK, (int)s.K) + 1024 - fixed;
      int sb = (int)((SMEM_CAP - fixed) / stage);
      if (sb > 4) sb = 4;
      const size_t smem = fixed + sb * stage;
#define PNN_DW(WP_, M_)                                                                                                \
  {                                                                                                                    \
    auto k = pnn_bwd_dw_tc_kernel<WP_, M_>;                                                                            \
    CTR_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                         \
    k<<<grid, NTHREADS, smem, st>>>(tg, to, e, dwt, (int)B, (int)F, (int)K, (int)N, (int)s.WX, ngroups, nslices, sb);  \
  }
      if (method == 0) {
        if (s.WP == 32) PNN_DW(32, 0) else if (s.WP == 64) PNN_DW(64, 0) else PNN_DW(128, 0)
      } else {
        if (s.WP == 32) PNN_DW(32, 1) else if (s.WP == 64) PNN_DW(64, 1) else PNN_DW(128, 1)
      }
#undef PNN_DW
      CTR_CHECK_LAUNCH("ctr_pnn_bwd(dw, wgmma)");
    }
  } else if (B > 0) {
    const size_t smem_dx = sizeof(float) * (size_t)(N + s.FK + s.K + s.WX);
    const size_t smem_dw = sizeof(float) * (size_t)(s.FK + s.K + SIMPLE_PC);
    CTR_UNSUPPORTED(smem_dx > SMEM_CAP, "ctr_pnn_bwd: N + F*K too large for the CUDA-core path");
    pnn_prep_kernel<<<grid_for((size_t)s.WX * N, 4096), 256, 0, st>>>(wlin, wprod, nullptr, ws, (int)F, (int)K, (int)N,
                                                                     method, (int)s.WX, (int)N, (int)s.WX, 0, 0);
    CTR_CHECK_LAUNCH("ctr_pnn_bwd(prep)");
    const int gdx = (int)(B < (int64_t)sms * 4 ? B : (int64_t)sms * 4);
    const int gx = (int)((s.WX + SIMPLE_PC - 1) / SIMPLE_PC), gy = (int)((N + 255) / 256);
    int gz = (int)((int64_t)sms * 4 / ((int64_t)gx * gy));
    if (gz < 1) gz = 1;
    if (gz > B) gz = (int)B;
    if (method == 0) {
      rc = set_smem((const void*)pnn_bwd_dx_simple_kernel<0>, smem_dx);
      if (rc) return rc;
      pnn_bwd_dx_simple_kernel<0><<<gdx, 256, smem_dx, st>>>(e, ws, out, g_out, d_e, (int)B, (int)F, (int)K, (int)N, (int)s.WX);
      CTR_CHECK_LAUNCH("ctr_pnn_bwd(dx, simple)");
      rc = set_smem((const void*)pnn_bwd_dw_simple_kernel<0>, smem_dw);
      if (rc) return rc;
      pnn_bwd_dw_simple_kernel<0><<<dim3(gx, gy, gz), 256, smem_dw, st>>>(e, out, g_out, dwt, (int)B, (int)F, (int)K, (int)N,
                                                                          (int)s.WX);
    } else {
      rc = set_smem((const void*)pnn_bwd_dx_simple_kernel<1>, smem_dx);
      if (rc) return rc;
      pnn_bwd_dx_simple_kernel<1><<<gdx, 256, smem_dx, st>>>(e, ws, out, g_out, d_e, (int)B, (int)F, (int)K, (int)N, (int)s.WX);
      CTR_CHECK_LAUNCH("ctr_pnn_bwd(dx, simple)");
      rc = set_smem((const void*)pnn_bwd_dw_simple_kernel<1>, smem_dw);
      if (rc) return rc;
      pnn_bwd_dw_simple_kernel<1><<<dim3(gx, gy, gz), 256, smem_dw, st>>>(e, out, g_out, dwt, (int)B, (int)F, (int)K, (int)N,
                                                                          (int)s.WX);
    }
    CTR_CHECK_LAUNCH("ctr_pnn_bwd(dw, simple)");
  }
  const size_t total = (size_t)s.FK * N + N + (method == 0 ? (size_t)N * F : (size_t)N * K * K);
  pnn_fold_kernel<<<grid_for(total, 4096), 256, 0, st>>>(dwt, wprod, d_wlin, d_wprod, d_bias, (int)F, (int)K, (int)N, method,
                                                        (int)s.WX);
  CTR_CHECK_LAUNCH("ctr_pnn_bwd(fold)");
  return CTR_OK;
}

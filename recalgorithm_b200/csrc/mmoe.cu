// MMoE expert-gate layer -- MMOE/mmoe.py:207-236: E expert dense(relu) layers, T softmax gates without bias, one gated sum
// per task.
//
//   a_e     = x . W_e + b_e          (B,H)   W_e = experts/expert_{e}/kernel (d,H), b_e = experts/expert_{e}/bias (H)
//   h_e     = relu(a_e)                      e = 0 .. E-1
//   p_t     = softmax_e(x . G_t)     (B,E)   G_t = gates/gate_{t}/kernel (d,E), no bias; t = 0 .. T-1
//   tower_t = sum_e p_t[e] h_e       (B,H)
// Backward, g_t = dL/dtower_t:  dp_t[e] = sum_h g_t h_e,  dlogit_t = p_t (dp_t - sum_e p_t dp_t),
//                               dz_e = (sum_t p_t[e] g_t) [a_e > 0],  dx = sum_e dz_e W_e^T + sum_t dlogit_t G_t^T,
//                               dW_e = x^T dz_e,  db_e = sum_b dz_e,  dG_t = x^T dlogit_t.
//
// H100 mapping: the row-chunk GEMMs of tc_ptx.cuh (rows namespace), as in the residual unit (csrc/residual_unit.cu): two
// consumer warpgroups of 64 samples + one TMA producer warp, wgmma kind tf32 with A in registers, 3xTF32, hidden-sized sums
// drained every 96 chained MMAs.  The weights are prepped once per call into the caller's workspace as tf32 hi | lo copies
// of one concatenated operand of R = E HP + GP units: the expert units e HP + h (H zero padded to HP, a multiple of HC =
// 32), then the GP = 32 gate columns t E + e (zero padded), each unit over DP = d rounded up to 32 / 64 / 96 / 128 inputs.
//   mmoe_fwd_wgmma_kernel     per 128-sample tile (and range of hidden chunks: a batch of fewer tiles than SMs splits
//                             the chunks over several CTAs): the gate logits x . [G_0 | .. | G_{T-1}] are one rows chunk; the softmax
//                             runs in registers over the quad of threads that shares a row (max subtracted, accurate expf)
//                             and the gates go to shared memory and to `gates`.  Then per hidden chunk, every expert's
//                             x . W_e[:, chunk] + b_e, relu in registers, and the T gated sums accumulated in registers and
//                             written straight to `towers`.  The (B, E, H) expert tensor never reaches global memory.
//   mmoe_bwd_dx_wgmma_kernel  per tile and (chunk, expert): a_e recomputed, gh_e = sum_t p_t[e] g_t, the dp_t[e] partials
//                             (reduced over the quad, summed per row in shared memory), dz_e = gh_e [a_e > 0] written to
//                             the workspace and fed from the accumulator registers to dx += dz_e . W_e[chunk]^T (hidden
//                             units in perm8 order).  After the last chunk: the softmax backward, dx += dlogit . G^T (one
//                             more hidden chunk: the gate columns), dlogit written to the workspace.
//   mmoe_bwd_dw_wgmma_kernel  one batch-sliced reduction over the workspace rows [dz_0 | .. | dz_{E-1} | dlogit] (pitch R)
//                             with B = x^T generated on chip (tc_ptx.cuh's batch_reduce, the residual unit's dW0 / db0
//                             mode): every dW_e with db_e as row sums, and every dG_t, one atomic per element per CTA.
// The rows of x, towers, gates and g are not 16-byte aligned in general (d = 82, H or E odd), so they are read and written
// with ordinary loads and stores; only the prepped weights and the workspace's dz | dlogit rows are TMA tensors.
//
// Tensor path (the only path): 1 <= d <= 128, 1 <= E <= MAX_E = 8, 1 <= H <= 1024, 1 <= T <= MAX_T = 4 (so T E <= GP = 32:
// the gate logits are one rows chunk), any B >= 0.  The T tower sums are T x 16 accumulator registers per thread, next to
// the 16 of the expert chunk and the 32 of its fragments; MAX_T = 4 keeps the forward well inside the register budget.
// Other shapes return CTR_ERR_UNSUPPORTED.
#include <math.h>

#include <algorithm>

#include "tc_ptx.cuh"

namespace ctr {
namespace mmoe {
using namespace ctr::tc;
using namespace ctr::tc::rows;

constexpr int TILE = NWG * WG_M;             // samples per CTA tile (forward, dx)
constexpr int MAX_E = 8, MAX_T = 4;
constexpr int GP = HC;                       // gate columns t E + e, zero padded to one rows chunk
constexpr int PLD = GP + 1;                  // pitch of the staged gate rows: rows g = 0..7 of a warp on distinct banks
static_assert(MAX_E * MAX_T <= GP, "the gate logits must fit one rows chunk");

// weight of concatenated unit n at input i (see the file header), 0 in the padding
__device__ __forceinline__ float unit_weight(const float* __restrict__ we, const float* __restrict__ wg, int n, int i, int d,
                                             int E, int H, int T, int HP) {
  if (i >= d) return 0.f;
  if (n < E * HP) {
    const int e = n / HP, h = n % HP;
    return h < H ? __ldg(we + ((size_t)e * d + i) * H + h) : 0.f;
  }
  const int c = n - E * HP;
  return c < T * E ? __ldg(wg + ((size_t)(c / E) * d + i) * E + c % E) : 0.f;
}

// Writes the tf32 hi | lo copies of the concatenated operand, one layout per blockIdx.y slot (2 R DP floats each):
//   0: rows operand [R][DP]    1: hidden operand [DP][R], units in perm8 order
__global__ void mmoe_prep_kernel(const float* __restrict__ we, const float* __restrict__ wg, float* __restrict__ dst, int d,
                                 int E, int H, int T, int DP, int HP, int R) {
  const int slot = blockIdx.y;
  const size_t total = (size_t)R * DP;
  float* o = dst + 2 * total * slot;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    int n, i;
    if (slot == 0) { n = (int)(idx / DP); i = (int)(idx % DP); }
    else { i = (int)(idx / R); n = perm8((int)(idx % R)); }
    store_split(o, total, idx, unit_weight(we, wg, n, i, d, E, H, T, HP));
  }
}

// ------------------------------------------------------------------------------------------------ shared device pieces
// In place: the gate logits of rows r0 (v[4c + x]) and r0 + 8 (v[4c + 2 + x]), columns 8c + 2t + x, become the softmax of
// each task's E columns; the padding columns become 0.  Every task's columns are spread over the quad of threads that
// shares the row, so the max and the sum are quad reductions.
__device__ __forceinline__ void gate_softmax(float (&v)[HC / 2], int E, int T, int t) {
  float p[HC / 2];
#pragma unroll
  for (int q = 0; q < HC / 2; ++q) p[q] = 0.f;
  for (int tt = 0; tt < T; ++tt) {
    float m[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int q = 0; q < HC / 2; ++q) {
      const int col = 8 * (q >> 2) + 2 * t + (q & 1);
      if (col >= tt * E && col < tt * E + E) m[(q >> 1) & 1] = fmaxf(m[(q >> 1) & 1], v[q]);
    }
    float s[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 1));
      m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 2));
    }
#pragma unroll
    for (int q = 0; q < HC / 2; ++q) {
      const int col = 8 * (q >> 2) + 2 * t + (q & 1);
      if (col >= tt * E && col < tt * E + E) {
        p[q] = expf(v[q] - m[(q >> 1) & 1]);
        s[(q >> 1) & 1] += p[q];
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      s[r] += __shfl_xor_sync(0xffffffffu, s[r], 1);
      s[r] += __shfl_xor_sync(0xffffffffu, s[r], 2);
    }
#pragma unroll
    for (int q = 0; q < HC / 2; ++q) {
      const int col = 8 * (q >> 2) + 2 * t + (q & 1);
      if (col >= tt * E && col < tt * E + E) p[q] = p[q] / s[(q >> 1) & 1];
    }
  }
#pragma unroll
  for (int q = 0; q < HC / 2; ++q) v[q] = p[q];
}

// ================================================================================================= forward
__host__ __device__ constexpr int fwd_smem_bytes(int DP, int SB) {
  return SB * stage_bytes(DP) + NWG * WG_M * (row_pitch(DP) + PLD) * 4 + 16 * SB;
}

template <int DP, int SB>
__global__ void __launch_bounds__(NTHREADS, 1)
mmoe_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_rows, const float* __restrict__ x,
                      const float* __restrict__ be, float* __restrict__ towers, float* __restrict__ gates, int B, int d,
                      int E, int H, int T, int HP, int nsplit) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int SBYTES = stage_bytes(DP), LD = row_pitch(DP);
  float* xs = reinterpret_cast<float*>(smem + SB * SBYTES);               // [2][64][LD]   x rows
  float* ps = xs + NWG * WG_M * LD;                                        // [2][64][PLD]  gates of those rows
  const uint32_t sbase = smem_u32(smem);
  Ring ring(smem_u32(ps + NWG * WG_M * PLD), SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_work = (B + TILE - 1) / TILE * nsplit, NC = HP / HC, R = E * HP + GP;
  ring.init();
  // ============================ TMA producer: the gate chunk, then per hidden chunk every expert's (hi, lo) ============
  if (producer_role(warp, lane, [&] {
        for (int wk = blockIdx.x; wk < n_work; wk += gridDim.x) {
          int j_beg, j_end;
          batch_slice(wk % nsplit, nsplit, NC, j_beg, j_end);
          Ring::Slot slot = ring.acquire(SBYTES);
          load_rows_operand<DP>(sbase + slot.stage * SBYTES, &tmap_rows, E * NC, R, slot.full);
          for (int j = j_beg; j < j_end; ++j)
            for (int e = 0; e < E; ++e) {
              slot = ring.acquire(SBYTES);
              load_rows_operand<DP>(sbase + slot.stage * SBYTES, &tmap_rows, e * NC + j, R, slot.full);
            }
        }
      }))
    return;

  // ============================ consumers ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3, tw = threadIdx.x & 127;
  const int r0 = w * 16 + g;
  float* xw = xs + wg * WG_M * LD;
  float* pw = ps + wg * WG_M * PLD;
  for (int wk = blockIdx.x; wk < n_work; wk += gridDim.x) {
    const int split = wk % nsplit;
    int j_beg, j_end;
    batch_slice(split, nsplit, NC, j_beg, j_end);
    const long long base = (long long)(wk / nsplit) * TILE + wg * WG_M;
    const bool v0 = base + r0 < B, v1 = base + r0 + 8 < B;
    stage_rows<DP>(xw, x, nullptr, base, B, d, tw);
    wg_bar_sync(1 + wg);
    {
      float p[HC / 2];
      gemm_rows<DP>(p, xw, r0, t, sbase + ring.wait() * SBYTES);
      ring.release(lane);
      gate_softmax(p, E, T, t);
#pragma unroll
      for (int q = 0; q < HC / 2; ++q) {
        const int col = 8 * (q >> 2) + 2 * t + (q & 1), r = r0 + 8 * ((q >> 1) & 1);
        pw[r * PLD + col] = p[q];
        if (split == 0 && col < T * E && base + r < B) gates[((size_t)(col / E) * B + base + r) * E + col % E] = p[q];
      }
    }
    __syncwarp();                             // rows r0 and r0 + 8 are this warp's own
    for (int j = j_beg; j < j_end; ++j) {
      float tow[MAX_T][HC / 2];
#pragma unroll
      for (int tt = 0; tt < MAX_T; ++tt)
#pragma unroll
        for (int q = 0; q < HC / 2; ++q) tow[tt][q] = 0.f;
      for (int e = 0; e < E; ++e) {
        float a[HC / 2];
        gemm_rows<DP>(a, xw, r0, t, sbase + ring.wait() * SBYTES);
        ring.release(lane);
        float pe[MAX_T][2];
#pragma unroll
        for (int tt = 0; tt < MAX_T; ++tt) {
          pe[tt][0] = tt < T ? pw[r0 * PLD + tt * E + e] : 0.f;
          pe[tt][1] = tt < T ? pw[(r0 + 8) * PLD + tt * E + e] : 0.f;
        }
#pragma unroll
        for (int q = 0; q < HC / 2; ++q) {
          const int col = j * HC + 8 * (q >> 2) + 2 * t + (q & 1);
          const float h = fmaxf(a[q] + (col < H ? __ldg(be + (size_t)e * H + col) : 0.f), 0.f);
#pragma unroll
          for (int tt = 0; tt < MAX_T; ++tt) tow[tt][q] = fmaf(pe[tt][(q >> 1) & 1], h, tow[tt][q]);
        }
      }
#pragma unroll
      for (int tt = 0; tt < MAX_T; ++tt) {
        if (tt >= T) break;
        float* o = towers + ((size_t)tt * B + base + r0) * H;
#pragma unroll
        for (int q = 0; q < HC / 2; ++q) {
          const int col = j * HC + 8 * (q >> 2) + 2 * t + (q & 1);
          const bool hi = (q >> 1) & 1;
          if (col < H && (hi ? v1 : v0)) o[(hi ? (size_t)8 * H : 0) + col] = tow[tt][q];
        }
      }
    }
    wg_bar_sync(1 + wg);                      // the rows may be restaged once every thread has read them
  }
}

// ================================================================================================= backward dx
__host__ __device__ constexpr int dx_smem_bytes(int DP, int SB) {
  return SB * stage_bytes(DP) + NWG * WG_M * (row_pitch(DP) + 2 * PLD) * 4 + 16 * SB;
}

template <int DP, int SB>
__global__ void __launch_bounds__(NTHREADS, 1)
mmoe_bwd_dx_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_rows, const __grid_constant__ CUtensorMap tmap_hidden,
                         const float* __restrict__ x, const float* __restrict__ be, const float* __restrict__ gates,
                         const float* __restrict__ g_towers, float* __restrict__ d_x, float* __restrict__ dzbuf, int B,
                         int d, int E, int H, int T, int HP) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int SBYTES = stage_bytes(DP), LD = row_pitch(DP);
  float* xs = reinterpret_cast<float*>(smem + SB * SBYTES);               // [2][64][LD]   x rows
  float* ps = xs + NWG * WG_M * LD;                                        // [2][64][PLD]  gates of those rows
  float* dps = ps + NWG * WG_M * PLD;                                      // [2][64][PLD]  dL/dgate, summed over chunks
  const uint32_t sbase = smem_u32(smem);
  Ring ring(smem_u32(dps + NWG * WG_M * PLD), SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_tiles = (B + TILE - 1) / TILE, NC = HP / HC, R = E * HP + GP;
  const int n_hidden = NC * E + 1;            // hidden GEMMs per tile: every (chunk, expert), then the gate columns
  ring.init();
  // ============================ TMA producer: per (chunk, expert) W_e^T and W_e, then the gate columns of G ===========
  if (producer_role(warp, lane, [&] {
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
          for (int j = 0; j < NC; ++j)
            for (int e = 0; e < E; ++e) {
              Ring::Slot slot = ring.acquire(SBYTES);
              load_rows_operand<DP>(sbase + slot.stage * SBYTES, &tmap_rows, e * NC + j, R, slot.full);
              slot = ring.acquire(SBYTES);
              load_hidden_operand<DP>(sbase + slot.stage * SBYTES, &tmap_hidden, e * NC + j, slot.full);
            }
          const Ring::Slot slot = ring.acquire(SBYTES);
          load_hidden_operand<DP>(sbase + slot.stage * SBYTES, &tmap_hidden, E * NC, slot.full);
        }
      }))
    return;

  // ============================ consumers ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3, tw = threadIdx.x & 127;
  const int r0 = w * 16 + g;
  float* xw = xs + wg * WG_M * LD;
  float* pw = ps + wg * WG_M * PLD;
  float* dpw = dps + wg * WG_M * PLD;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long base = (long long)tile * TILE + wg * WG_M;
    const bool v0 = base + r0 < B, v1 = base + r0 + 8 < B;
    stage_rows<DP>(xw, x, nullptr, base, B, d, tw);
    for (int idx = tw; idx < WG_M * GP; idx += 128) {
      const int r = idx / GP, c = idx % GP;
      pw[r * PLD + c] = (c < T * E && base + r < B) ? __ldg(gates + ((size_t)(c / E) * B + base + r) * E + c % E) : 0.f;
      dpw[r * PLD + c] = 0.f;
    }
    wg_bar_sync(1 + wg);
    float* dz0 = dzbuf + (size_t)(base + r0) * R;
    float acc[DP / 2], dacc[DP / 2];
#pragma unroll
    for (int q = 0; q < DP / 2; ++q) { acc[q] = 0.f; dacc[q] = 0.f; }
    int i = 0;                                // hidden GEMM index of the accumulation chains
    for (int j = 0; j < NC; ++j) {
      for (int e = 0; e < E; ++e, ++i) {
        float a[HC / 2];
        gemm_rows<DP>(a, xw, r0, t, sbase + ring.wait() * SBYTES);
        ring.release(lane);
#pragma unroll
        for (int q = 0; q < HC / 2; ++q) {    // h_e, and h_e > 0 exactly where a_e > 0
          const int col = j * HC + 8 * (q >> 2) + 2 * t + (q & 1);
          a[q] = fmaxf(a[q] + (col < H ? __ldg(be + (size_t)e * H + col) : 0.f), 0.f);
        }
        float gh[HC / 2];
#pragma unroll
        for (int q = 0; q < HC / 2; ++q) gh[q] = 0.f;
        for (int tt = 0; tt < T; ++tt) {
          const float p0 = pw[r0 * PLD + tt * E + e], p1 = pw[(r0 + 8) * PLD + tt * E + e];
          const float* gt = g_towers + ((size_t)tt * B + base + r0) * H;
          float s[2] = {0.f, 0.f};
#pragma unroll
          for (int q = 0; q < HC / 2; ++q) {
            const int col = j * HC + 8 * (q >> 2) + 2 * t + (q & 1);
            const bool hi = (q >> 1) & 1;
            const float gv = col < H && (hi ? v1 : v0) ? __ldg(gt + (hi ? (size_t)8 * H : 0) + col) : 0.f;
            gh[q] = fmaf(hi ? p1 : p0, gv, gh[q]);
            s[hi] = fmaf(gv, a[q], s[hi]);
          }
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            s[r] += __shfl_xor_sync(0xffffffffu, s[r], 1);
            s[r] += __shfl_xor_sync(0xffffffffu, s[r], 2);
          }
          if (t == 0) {
            dpw[r0 * PLD + tt * E + e] += s[0];
            dpw[(r0 + 8) * PLD + tt * E + e] += s[1];
          }
        }
#pragma unroll
        for (int q = 0; q < HC / 2; ++q) gh[q] = a[q] > 0.f ? gh[q] : 0.f;
#pragma unroll
        for (int c = 0; c < HC / 8; ++c) {
          const int col = e * HP + j * HC + 8 * c + 2 * t;
          if (v0) *reinterpret_cast<float2*>(dz0 + col) = make_float2(gh[4 * c], gh[4 * c + 1]);
          if (v1) *reinterpret_cast<float2*>(dz0 + (size_t)8 * R + col) = make_float2(gh[4 * c + 2], gh[4 * c + 3]);
        }
        uint32_t hh[HC / 8][4], hl[HC / 8][4];
        acc_to_a(gh, hh, hl);
        gemm_hidden<DP>(dacc, hh, hl, sbase + ring.wait() * SBYTES, chain_first(i, CHAIN));
        ring.release(lane);
        if (chain_last(i, n_hidden, CHAIN)) chain_drain(acc, dacc);
      }
    }
    __syncwarp();                             // the dp sums of rows r0 and r0 + 8 were added by this warp's t = 0 lanes
    // softmax backward: dlogit[col] = p (dp - sum_e p dp) over the E columns of col's task
    float dl[HC / 2];
#pragma unroll
    for (int q = 0; q < HC / 2; ++q) {
      const int col = 8 * (q >> 2) + 2 * t + (q & 1), r = r0 + 8 * ((q >> 1) & 1);
      dl[q] = 0.f;
      if (col < T * E) {
        const int c0 = col / E * E;
        float sum = 0.f;
        for (int e = 0; e < E; ++e) sum = fmaf(pw[r * PLD + c0 + e], dpw[r * PLD + c0 + e], sum);
        dl[q] = pw[r * PLD + col] * (dpw[r * PLD + col] - sum);
      }
    }
#pragma unroll
    for (int c = 0; c < HC / 8; ++c) {
      const int col = E * HP + 8 * c + 2 * t;
      if (v0) *reinterpret_cast<float2*>(dz0 + col) = make_float2(dl[4 * c], dl[4 * c + 1]);
      if (v1) *reinterpret_cast<float2*>(dz0 + (size_t)8 * R + col) = make_float2(dl[4 * c + 2], dl[4 * c + 3]);
    }
    {
      uint32_t hh[HC / 8][4], hl[HC / 8][4];
      acc_to_a(dl, hh, hl);
      gemm_hidden<DP>(dacc, hh, hl, sbase + ring.wait() * SBYTES, chain_first(i, CHAIN));
      ring.release(lane);
      chain_drain(acc, dacc);                 // i = n_hidden - 1 ends the last chain
    }
#pragma unroll
    for (int c = 0; c < DP / 8; ++c) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int k = 8 * c + 2 * t + e;
        if (k < d) {
          if (v0) d_x[(size_t)(base + r0) * d + k] = acc[4 * c + e];
          if (v1) d_x[(size_t)(base + r0 + 8) * d + k] = acc[4 * c + 2 + e];
        }
      }
    }
    wg_bar_sync(1 + wg);
  }
}

// ================================================================================================= backward dW
__host__ __device__ constexpr int dw_smem_bytes(int DP, int SB) { return SB * (2 * DP * 128 + DW_BC * DW_NC * 4 + 16); }

// P = the workspace rows [dz_0 | .. | dz_{E-1} | dlogit] (B, R), Q = x: row n < E HP of the result is dW_e[:, h]
// (n = e HP + h) with db_e[h] its sum over the batch, row E HP + t E + e is dG_t[:, e].
template <int DP>
__global__ void __launch_bounds__(NTHREADS, 1)
mmoe_bwd_dw_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_p, const float* __restrict__ x, float* __restrict__ d_we,
                         float* __restrict__ d_be, float* __restrict__ d_wg, int B, int d, int E, int H, int T, int HP,
                         int ngroups, int nslices, int SB) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int qt_bytes = 2 * DP * 128;                    // Q^T tiles [DP x 32 samples] (hi | lo), 128B-swizzled
  constexpr int p_floats = DW_BC * DW_NC;                   // one P chunk [32 samples x 128 units]
  uint8_t* qts = smem;
  float* ps = reinterpret_cast<float*>(smem + SB * qt_bytes);
  Ring ring(smem_u32(ps + SB * p_floats), SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int group = blockIdx.x % ngroups;
  int c_beg, c_end;
  batch_slice(blockIdx.x / ngroups, nslices, (B + DW_BC - 1) / DW_BC, c_beg, c_end);
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

  // ============================ consumers: B = x^T generated on chip, A = P^T ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3;
  float rsum[2] = {0.f, 0.f};                               // sum_b of this thread's two rows (db_e for expert units)
  const int nl0 = wg * WG_M + w * 16 + g;                   // this thread's A rows: units n0 + nl0 (+8)
  float acc[DP / 2];
  batch_reduce<DP>(
      acc, ring, qts, c_beg, c_end, B, lane, nl0, [](int) {},
      [&](int k, int b0, int b) { return k < d ? __ldg(x + (size_t)(b0 + b) * d + k) : 0.f; },
      [&](int s, int b, int nl) {
        const float v = ps[(size_t)s * p_floats + b * DW_NC + nl];
        rsum[nl == nl0 ? 0 : 1] += v;
        return v;
      });
  if (c_end <= c_beg) return;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int n = n0 + nl0 + 8 * r;
    float* dst = nullptr;                                   // element k of this row: dst[k * stride]
    size_t stride = 0;
    if (n < E * HP) {
      const int e = n / HP, h = n % HP;
      if (h < H) { dst = d_we + (size_t)e * d * H + h; stride = H; }
    } else if (n - E * HP < T * E) {
      const int c = n - E * HP;
      dst = d_wg + (size_t)(c / E) * d * E + c % E;
      stride = E;
    }
#pragma unroll
    for (int cc = 0; cc < DP / 8; ++cc) {
#pragma unroll
      for (int xx = 0; xx < 2; ++xx) {
        const int k = 8 * cc + 2 * t + xx;
        if (dst != nullptr && k < d) atomicAdd(dst + (size_t)k * stride, acc[4 * cc + 2 * r + xx]);
      }
    }
    float v = rsum[r];
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    if (t == 0 && n < E * HP && n % HP < H) atomicAdd(d_be + (size_t)(n / HP) * H + n % HP, v);
  }
}

}  // namespace mmoe
}  // namespace ctr

// ------------------------------------------------------------------------------------------------ host
using namespace ctr;
using namespace ctr::mmoe;

namespace {

struct MmShape {
  int DP;
  int64_t HP, R;
  int64_t slot_floats;             // one prepped layout: hi | lo copies of [R][DP] or [DP][R]
  int64_t dz_offset;               // workspace byte offset of the dz | dlogit rows (B, R) (backward)
  int64_t fwd_bytes, bwd_bytes;
};

MmShape shape_of(int64_t B, int64_t d, int64_t E, int64_t H) {
  MmShape s;
  s.DP = dp_class(d);
  s.HP = pad_to(H, HC);
  s.R = E * s.HP + GP;
  s.slot_floats = 2 * s.R * s.DP;
  s.fwd_bytes = pad_to(s.slot_floats * (int64_t)sizeof(float), 128);
  s.dz_offset = pad_to(2 * s.slot_floats * (int64_t)sizeof(float), 128);
  s.bwd_bytes = s.dz_offset + pad_to(B * s.R * (int64_t)sizeof(float), 128);
  return s;
}

int check_shape(const char* fn, int64_t B, int64_t d, int64_t E, int64_t H, int64_t T) {
  CTR_REQUIRE(B >= 0 && d >= 1 && E >= 1 && H >= 1 && T >= 1, "%s: bad sizes B=%lld d=%lld E=%lld H=%lld T=%lld", fn,
              (long long)B, (long long)d, (long long)E, (long long)H, (long long)T);
  CTR_UNSUPPORTED(d > 128, "%s: unsupported input width d=%lld (the tensor-core kernels take d <= 128)", fn, (long long)d);
  CTR_UNSUPPORTED(E > MAX_E, "%s: unsupported num_experts E=%lld (the tensor-core kernels take E <= %d)", fn, (long long)E,
                  MAX_E);
  CTR_UNSUPPORTED(H > 1024, "%s: unsupported expert_hidden_units H=%lld (the tensor-core kernels take H <= 1024)", fn,
                  (long long)H);
  CTR_UNSUPPORTED(T > MAX_T, "%s: unsupported num_tasks T=%lld (the tensor-core kernels take T <= %d)", fn, (long long)T,
                  MAX_T);
  CTR_UNSUPPORTED(B > 0x7fffff00LL, "%s: batch too large (B=%lld)", fn, (long long)B);
  return CTR_OK;
}

int prep(const char* what, const float* we, const float* wg, float* ws, int64_t d, int64_t E, int64_t H, int64_t T,
         const MmShape& s, int nslots, cudaStream_t st) {
  return launch(what, mmoe_prep_kernel, dim3(capped_grid((s.R * s.DP + 255) / 256, 1024), nslots), 256, 0, st, we, wg, ws,
                (int)d, (int)E, (int)H, (int)T, s.DP, (int)s.HP, (int)s.R);
}

}  // namespace

extern "C" int ctr_mmoe_workspace_bytes(int64_t B, int64_t d, int64_t E, int64_t H, int64_t T, int64_t* bytes) {
  int rc = check_shape("ctr_mmoe_workspace_bytes", B, d, E, H, T);
  if (rc) return rc;
  CTR_REQUIRE(bytes != nullptr, "ctr_mmoe_workspace_bytes: null argument");
  *bytes = shape_of(B, d, E, H).bwd_bytes;
  return CTR_OK;
}

extern "C" int ctr_mmoe_fwd(const float* x, const float* w_experts, const float* b_experts, const float* w_gates, int64_t B,
                            int64_t d, int64_t E, int64_t H, int64_t T, float* towers, float* gates, void* workspace,
                            int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_mmoe_fwd";
  int rc = check_shape(fn, B, d, E, H, T);
  if (rc) return rc;
  CTR_REQUIRE(x && w_experts && b_experts && w_gates && towers && gates, "ctr_mmoe_fwd: null argument");
  const MmShape s = shape_of(B, d, E, H);
  rc = check_workspace(fn, "ctr_mmoe_workspace_bytes with B = 0", workspace, workspace_bytes, s.fwd_bytes);
  if (rc) return rc;
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  float* ws = static_cast<float*>(workspace);
  if ((rc = prep("ctr_mmoe_fwd(prep)", w_experts, w_gates, ws, d, E, H, T, s, 1, st))) return rc;
  CUtensorMap mr;
  if ((rc = encode_rows_operand(fn, &mr, ws, s.DP, s.R))) return rc;
  // Small batches split the hidden chunks of each tile over several CTAs (each recomputes the tile's gates) to fill the SMs.
  const int sms = sm_count();
  const int64_t n_tiles = (B + TILE - 1) / TILE;
  const int nsplit = (int)std::max<int64_t>(1, std::min<int64_t>(sms / n_tiles, s.HP / HC));
  const int grid = capped_grid(n_tiles * nsplit, sms);
  return with_const<32, 64, 96, 128>(s.DP, [&](auto DP) {
    constexpr int SB = 4;
    static_assert(fwd_smem_bytes(DP, SB) + 1024 <= SMEM_CAP, "forward shared memory");
    return launch("ctr_mmoe_fwd(wgmma)", mmoe_fwd_wgmma_kernel<DP, SB>, grid, NTHREADS, fwd_smem_bytes(DP, SB) + 1024, st,
                  mr, x, b_experts, towers, gates, (int)B, (int)d, (int)E, (int)H, (int)T, (int)s.HP, nsplit);
  });
}

extern "C" int ctr_mmoe_bwd(const float* x, const float* w_experts, const float* b_experts, const float* w_gates,
                            const float* gates, const float* g_towers, int64_t B, int64_t d, int64_t E, int64_t H, int64_t T,
                            float* d_x, float* d_w_experts, float* d_b_experts, float* d_w_gates, void* workspace,
                            int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_mmoe_bwd";
  int rc = check_shape(fn, B, d, E, H, T);
  if (rc) return rc;
  CTR_REQUIRE(x && w_experts && b_experts && w_gates && gates && g_towers && d_x && d_w_experts && d_b_experts && d_w_gates,
              "ctr_mmoe_bwd: null argument");
  const MmShape s = shape_of(B, d, E, H);
  rc = check_workspace(fn, "ctr_mmoe_workspace_bytes", workspace, workspace_bytes, s.bwd_bytes);
  if (rc) return rc;
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(d_w_experts, 0, sizeof(float) * (size_t)(E * d * H), st));
  CTR_CUDA(cudaMemsetAsync(d_b_experts, 0, sizeof(float) * (size_t)(E * H), st));
  CTR_CUDA(cudaMemsetAsync(d_w_gates, 0, sizeof(float) * (size_t)(T * d * E), st));
  if (B == 0) return CTR_OK;
  float* ws = static_cast<float*>(workspace);
  float* dzbuf = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + s.dz_offset);
  if ((rc = prep("ctr_mmoe_bwd(prep)", w_experts, w_gates, ws, d, E, H, T, s, 2, st))) return rc;
  CUtensorMap mr, mh, mdz;
  if ((rc = encode_rows_operand(fn, &mr, ws, s.DP, s.R)) ||
      (rc = encode_hidden_operand(fn, &mh, ws + s.slot_floats, s.DP, s.R)) ||
      (rc = encode_2d(fn, &mdz, dzbuf, s.R, B, DW_NC, DW_BC, CU_TENSOR_MAP_SWIZZLE_NONE)))
    return rc;
  const int sms = sm_count();
  const int grid = capped_grid((B + TILE - 1) / TILE, sms);
  const int ngroups = (int)((s.R + DW_NC - 1) / DW_NC);
  const int nslices = batch_slices(sms, ngroups, (B + DW_BC - 1) / DW_BC);
  return with_const<32, 64, 96, 128>(s.DP, [&](auto DP) {
    constexpr int SB = DP == 128 ? 3 : 4;
    static_assert(dx_smem_bytes(DP, SB) + 1024 <= SMEM_CAP, "dx shared memory");
    if (int r = launch("ctr_mmoe_bwd(dx, wgmma)", mmoe_bwd_dx_wgmma_kernel<DP, SB>, grid, NTHREADS,
                       dx_smem_bytes(DP, SB) + 1024, st, mr, mh, x, b_experts, gates, g_towers, d_x, dzbuf, (int)B, (int)d,
                       (int)E, (int)H, (int)T, (int)s.HP))
      return r;
    const int sb = stages_that_fit(1024, dw_smem_bytes(DP, 1));
    return launch("ctr_mmoe_bwd(dw, wgmma)", mmoe_bwd_dw_wgmma_kernel<DP>, ngroups * nslices, NTHREADS,
                  dw_smem_bytes(DP, sb) + 1024, st, mdz, x, d_w_experts, d_b_experts, d_w_gates, (int)B, (int)d, (int)E,
                  (int)H, (int)T, (int)s.HP, ngroups, nslices, sb);
  });
}

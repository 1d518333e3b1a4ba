// PLE expert-gate blocks -- PLE/extraction_network.py:4-85 (the extraction network) and PLE/ple.py:185-226 (the final
// layer).  Both are one computation over E = sum_t n_t + S experts and G gates:
//
//   a_e   = x . W_e + b_e,  h_e = relu(a_e)          W_e (d,H), b_e (H); experts [task 0 .. task T-1, shared]
//   z     = x . Gcat                         (B,GC)  Gcat = [gate_0 | .. | gate_{T-1} (| all_gate)], no bias
//   p_g   = softmax over gate g's columns            gate t < T: [task t's n_t experts, the S shared ones]; all_gate: all E
//   out_o = sum_{g -> o} sum_j p_g[j] h_{e(g,j)}     final layer: O = T outputs, gate t -> output t;
//                                                    extraction network: O = 1, every gate -> output 0 (the add_n)
// Backward, g_o = dL/dout_o:  dp_g[j] = <g_o, h_{e(g,j)}>,  dlogit_g = p_g (dp_g - sum_j p_g[j] dp_g[j]),
//   dz_e = (sum_o c_o[e] g_o) [a_e > 0] with c_o[e] the sum of the p_g[j] that point at e for the gates g -> o,
//   dx = sum_e dz_e W_e^T + dlogit Gcat^T,  dW_e = x^T dz_e,  db_e = sum_b dz_e,  dGcat = x^T dlogit.
//
// H100 mapping (3xTF32 wgmma, one TMA producer warp, two consumer warpgroups).  The weights are prepped once per call into
// the caller's workspace as tf32 hi | lo copies of one concatenated operand of R = E HP + GP units: expert e's units
// e HP + h (H zero padded to HP, a multiple of PC = 64), then the GC gate columns (zero padded to GP, a multiple of 64).
//   ple_fwd_wgmma_kernel     per 64-sample tile: the tile's x rows (width up to 512) are staged once in shared memory and
//                            both warpgroups read them; they take the two 32-unit halves of every 64-unit ring stage, so
//                            their outputs never overlap.  A stage holds [64 units x 32 inputs] (16 KB): the rows GEMMs are
//                            K-sliced, so the ring depth does not depend on d.  First the gate logits (GP / 64 unit
//                            pairs) into a shared [64 x GC] table, the per-gate softmax in place (one thread per row and
//                            gate, max subtracted, accurate expf) and out to `gates`; then per 64 hidden units, every
//                            expert's GEMM, bias and relu in registers and the O gated sums accumulated in registers and
//                            written to `out`.  The (B, E, H) expert tensor never reaches global memory.  A batch of fewer
//                            tiles than SMs splits the hidden units of each tile over several CTAs.
//   ple_bwd_dz_wgmma_kernel  per 64-sample tile and expert: a_e recomputed, dz_e = (sum_o c_o[e] g_o) [a_e > 0] written to
//                            the workspace, and <g_o, h_e> summed per row into a shared dp table.  Then the softmax
//                            backward, dlogit written to the workspace next to dz: rows [dz_0 | .. | dz_{E-1} | dlogit].
//   ple_bwd_dx_wgmma_kernel  dx = [dz | dlogit] . [W | Gcat]^T: per 128-sample tile and N-wide slice of d, a K-sliced GEMM
//                            over the R units, both operands TMA-staged (the workspace rows and the hidden-layout prep).
//   ple_bwd_dw_wgmma_kernel  one batch-sliced reduction over the workspace rows with x^T generated on chip (tc_ptx.cuh's
//                            batch_reduce), one grid dimension per N-wide slice of d: every dW_e with db_e, and dGcat.
// x, out, gates and g are read and written with ordinary loads and stores (d, H and GC are arbitrary); the prepped weights
// and the workspace rows are TMA tensors.
//
// Bounds: 1 <= d <= 512, 1 <= H <= 512, 1 <= T <= 4, n_t >= 1, S >= 1, E <= 64 and GC <= 160 (the shared gate table
// next to a 512-wide x tile), any B >= 0.  Other shapes return CTR_ERR_UNSUPPORTED.
#include <math.h>

#include <algorithm>

#include "tc_ptx.cuh"

namespace ctr {
namespace ple {
using namespace ctr::tc;
using namespace ctr::tc::rows;

constexpr int TM = WG_M;                     // samples per forward / dz tile: both warpgroups share the tile's rows
constexpr int PC = 2 * HC;                   // units per ring stage: one 32-unit half per warpgroup
constexpr int SBYTES = 2 * PC * KB * 4;      // one stage: [64 units x 32 inputs], hi then lo
constexpr int MAX_D = 512, MAX_H = 512, MAX_T = 4, MAX_E = 64, MAX_GC = 160;
constexpr int DX_TILE = NWG * WG_M;          // samples per dx tile
// 32-input slices per accumulation chain (4 k-steps x 3 = 12 MMAs each).  The tensor core truncates as it accumulates; with
// 96-MMA chains the widest inputs missed the fp32 bars by up to 1.2x (the softmax turns a gate logit's absolute error into
// the gate's relative error).  The row GEMMs drain every slice, the dx GEMM every two (its drain is 64 adds per thread).
constexpr int KCHAIN = 1, DX_KCHAIN = 2;

// The gate structure of one call.  Experts: task t's at e0[t] .. e0[t] + n[t], the shared ones at ES .. ES + S.  Gate
// g < T has columns c0[g] .. c0[g] + n[g] + S over [task g's experts, shared]; gate T (extraction network only) has
// columns c0[T] .. c0[T] + E over all experts in order.
struct Gates {
  int T, S, E, ES, G, O, GC;
  int n[MAX_T], e0[MAX_T], c0[MAX_T + 1];
};

__host__ __device__ __forceinline__ int gate_len(const Gates& q, int g) { return g < q.T ? q.n[g] + q.S : q.E; }
__host__ __device__ __forceinline__ int gate_out(const Gates& q, int g) { return q.O == 1 ? 0 : g; }
// expert of column j of gate g
__host__ __device__ __forceinline__ int gate_expert(const Gates& q, int g, int j) {
  return g == q.T ? j : j < q.n[g] ? q.e0[g] + j : q.ES + j - q.n[g];
}
// column of expert e within gate g, or -1
__host__ __device__ __forceinline__ int gate_pos(const Gates& q, int g, int e) {
  if (g == q.T) return e;
  if (e >= q.e0[g] && e < q.e0[g] + q.n[g]) return e - q.e0[g];
  return e >= q.ES ? q.n[g] + e - q.ES : -1;
}
// c_o[e] of one row from its gate probabilities prow (GC columns)
__device__ __forceinline__ float coef(const Gates& q, const float* prow, int o, int e) {
  float c = 0.f;
  for (int g = 0; g < q.G; ++g) {
    const int j = gate_pos(q, g, e);
    if (gate_out(q, g) == o && j >= 0) c += prow[q.c0[g] + j];
  }
  return c;
}
// Slot of <g_o, h_e> in a row of the dp table: the final layer keeps one per gate column (gate o's column of e, or -1
// when e is not in gate o); the extraction network has one output, so one per expert.
__device__ __forceinline__ int dp_slot(const Gates& q, int o, int e) {
  if (q.O == 1) return e;
  const int j = gate_pos(q, o, e);
  return j >= 0 ? q.c0[o] + j : -1;
}

// weight of concatenated unit n at input i (see the file header), 0 in the padding
__device__ __forceinline__ float unit_weight(const float* __restrict__ we, const float* __restrict__ wg, int n, int i, int d,
                                             int E, int H, int GC, int HP) {
  if (i >= d) return 0.f;
  if (n < E * HP) {
    const int e = n / HP, h = n % HP;
    return h < H ? __ldg(we + ((size_t)e * d + i) * H + h) : 0.f;
  }
  const int c = n - E * HP;
  return c < GC ? __ldg(wg + (size_t)i * GC + c) : 0.f;
}

// Writes the tf32 hi | lo copies of the concatenated operand, one layout per blockIdx.y:
//   0: rows operand [R][DP] at dst_rows     1: hidden operand [DH][R] at dst_hidden (backward)
__global__ void ple_prep_kernel(const float* __restrict__ we, const float* __restrict__ wg, float* __restrict__ dst_rows,
                                float* __restrict__ dst_hidden, int d, int E, int H, int GC, int DP, int DH, int HP, int R) {
  const bool rows = blockIdx.y == 0;
  const size_t total = (size_t)R * (rows ? DP : DH);
  float* o = rows ? dst_rows : dst_hidden;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int n = rows ? (int)(idx / DP) : (int)(idx % R), i = rows ? (int)(idx % DP) : (int)(idx / R);
    const float v = unit_weight(we, wg, n, i, d, E, H, GC, HP), hi = tf32_rna(v);
    o[idx] = hi;                              // hi | lo, with lo rounded to tf32 too (the tensor core would truncate it)
    o[total + idx] = tf32_rna(v - hi);
  }
}

// ------------------------------------------------------------------------------------------------ shared device pieces
// TMA loads of one stage: units u0 .. u0 + 63, inputs 32 kb .. 32 kb + 31, hi then lo, from the [2 R][DP] rows map.
__device__ __forceinline__ void load_stage(uint32_t dst, const CUtensorMap* map, int u0, int kb, int R, uint32_t bar) {
  tma_load_2d(dst, map, kb * KB, u0, bar);
  tma_load_2d(dst + PC * 128, map, kb * KB, R + u0, bar);
}

// D[64 x HC] = X[64 x DP] . B over the next nk ring stages: X = the tile's staged rows (pitch ldx), B = this warpgroup's
// 32-unit half of each stage.  One 32-input slice (4 k-steps) per stage; chains of KCHAIN slices drained into d.
__device__ __forceinline__ void gemm_ks(float (&d)[HC / 2], const float* xs, int ldx, int nk, int r0, int t, int lane,
                                        int wg, Ring& ring, uint32_t sbase) {
  float dacc[HC / 2];
#pragma unroll
  for (int q = 0; q < HC / 2; ++q) { d[q] = 0.f; dacc[q] = 0.f; }
  for (int kb = 0; kb < nk; ++kb) {
    const uint32_t st = sbase + ring.wait() * SBYTES + wg * HC * 128;
    const uint64_t bhi = gmma_desc_kmajor(st, 128), blo = gmma_desc_kmajor(st + PC * 128, 128);
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      float a[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) a[q] = xs[(r0 + 8 * (q & 1)) * ldx + kb * KB + 8 * ks + t + 4 * (q >> 1)];
      tf32_split(a, ah[ks], al[ks]);
    }
    const bool start = chain_first(kb, KCHAIN);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) mma_3xtf32<HC>(dacc, ah[ks], al[ks], bhi, blo, (uint64_t)(2 * ks), (start && ks == 0) ? 0 : 1);
    wgmma_commit();
    wgmma_wait_keep(ah, al);
    ring.release(lane);
    if (chain_last(kb, nk, KCHAIN)) chain_drain(d, dacc);
  }
}

// Stages the tile's 64 rows of x (B,d), zero padded to DP columns and past B, with all 256 consumer threads.
__device__ __forceinline__ void stage_tile(float* xs, int ldx, const float* __restrict__ x, long long base, int B, int d,
                                           int DP) {
  for (int idx = threadIdx.x; idx < TM * DP; idx += NWG * 128) {
    const int r = idx / DP, c = idx % DP;
    xs[r * ldx + c] = (c < d && base + r < B) ? __ldg(x + (size_t)(base + r) * d + c) : 0.f;
  }
}

__host__ __device__ constexpr int tile_bytes(int DP, int GC, int SB) {
  return SB * SBYTES + TM * (DP + 4) * 4 + TM * (GC + 1) * 4 + 16 * SB;
}

// ================================================================================================= forward
__global__ void __launch_bounds__(NTHREADS, 1)
ple_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_rows, const __grid_constant__ Gates q,
                     const float* __restrict__ x, const float* __restrict__ be, float* __restrict__ out,
                     float* __restrict__ gates, int B, int d, int H, int DP, int HP, int GP, int nsplit, int SB) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  const int ldx = DP + 4, ldp = q.GC + 1, nk = DP / KB, NJ = HP / PC, R = q.E * HP + GP;
  float* xs = reinterpret_cast<float*>(smem + SB * SBYTES);               // [64][ldx]   x rows
  float* ps = xs + TM * ldx;                                               // [64][ldp]   gate logits, then probabilities
  const uint32_t sbase = smem_u32(smem);
  Ring ring(smem_u32(ps + TM * ldp), SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_work = (B + TM - 1) / TM * nsplit;
  ring.init();
  // ============================ TMA producer: the gate unit pairs, then per 64 hidden units every expert ============
  if (producer_role(warp, lane, [&] {
        for (int wk = blockIdx.x; wk < n_work; wk += gridDim.x) {
          int j_beg, j_end;
          batch_slice(wk % nsplit, nsplit, NJ, j_beg, j_end);
          for (int gp = 0; gp < GP / PC; ++gp)
            for (int kb = 0; kb < nk; ++kb) {
              const Ring::Slot slot = ring.acquire(SBYTES);
              load_stage(sbase + slot.stage * SBYTES, &tmap_rows, q.E * HP + gp * PC, kb, R, slot.full);
            }
          for (int j = j_beg; j < j_end; ++j)
            for (int e = 0; e < q.E; ++e)
              for (int kb = 0; kb < nk; ++kb) {
                const Ring::Slot slot = ring.acquire(SBYTES);
                load_stage(sbase + slot.stage * SBYTES, &tmap_rows, e * HP + j * PC, kb, R, slot.full);
              }
        }
      }))
    return;

  // ============================ consumers ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3;
  const int r0 = w * 16 + g;
  for (int wk = blockIdx.x; wk < n_work; wk += gridDim.x) {
    const int split = wk % nsplit;
    int j_beg, j_end;
    batch_slice(split, nsplit, NJ, j_beg, j_end);
    const long long base = (long long)(wk / nsplit) * TM;
    const bool v0 = base + r0 < B, v1 = base + r0 + 8 < B;
    stage_tile(xs, ldx, x, base, B, d, DP);
    consumers_bar();
    for (int gp = 0; gp < GP / PC; ++gp) {
      float z[HC / 2];
      gemm_ks(z, xs, ldx, nk, r0, t, lane, wg, ring, sbase);
#pragma unroll
      for (int k = 0; k < HC / 2; ++k) {
        const int col = gp * PC + wg * HC + 8 * (k >> 2) + 2 * t + (k & 1), r = r0 + 8 * ((k >> 1) & 1);
        if (col < q.GC) ps[r * ldp + col] = z[k];
      }
    }
    consumers_bar();
    for (int idx = threadIdx.x; idx < TM * q.G; idx += NWG * 128) {     // per-gate softmax, one thread per (row, gate)
      const int r = idx / q.G, gi = idx % q.G, len = gate_len(q, gi);
      float* p = ps + r * ldp + q.c0[gi];
      float m = -INFINITY, s = 0.f;
      for (int j = 0; j < len; ++j) m = fmaxf(m, p[j]);
      for (int j = 0; j < len; ++j) { p[j] = expf(p[j] - m); s += p[j]; }
      for (int j = 0; j < len; ++j) {
        p[j] = p[j] / s;
        if (split == 0 && base + r < B) gates[(size_t)(base + r) * q.GC + q.c0[gi] + j] = p[j];
      }
    }
    consumers_bar();
    for (int j = j_beg; j < j_end; ++j) {
      float acc[MAX_T][HC / 2];
#pragma unroll
      for (int o = 0; o < MAX_T; ++o)
#pragma unroll
        for (int k = 0; k < HC / 2; ++k) acc[o][k] = 0.f;
      for (int e = 0; e < q.E; ++e) {
        float a[HC / 2];
        gemm_ks(a, xs, ldx, nk, r0, t, lane, wg, ring, sbase);
        float pe[MAX_T][2];
#pragma unroll
        for (int o = 0; o < MAX_T; ++o) {
          pe[o][0] = o < q.O ? coef(q, ps + r0 * ldp, o, e) : 0.f;
          pe[o][1] = o < q.O ? coef(q, ps + (r0 + 8) * ldp, o, e) : 0.f;
        }
#pragma unroll
        for (int k = 0; k < HC / 2; ++k) {
          const int col = j * PC + wg * HC + 8 * (k >> 2) + 2 * t + (k & 1);
          const float h = fmaxf(a[k] + (col < H ? __ldg(be + (size_t)e * H + col) : 0.f), 0.f);
#pragma unroll
          for (int o = 0; o < MAX_T; ++o) acc[o][k] = fmaf(pe[o][(k >> 1) & 1], h, acc[o][k]);
        }
      }
#pragma unroll
      for (int o = 0; o < MAX_T; ++o) {
        if (o >= q.O) break;
        float* dst = out + ((size_t)o * B + base + r0) * H;
#pragma unroll
        for (int k = 0; k < HC / 2; ++k) {
          const int col = j * PC + wg * HC + 8 * (k >> 2) + 2 * t + (k & 1);
          const bool hi = (k >> 1) & 1;
          if (col < H && (hi ? v1 : v0)) dst[(hi ? (size_t)8 * H : 0) + col] = acc[o][k];
        }
      }
    }
    consumers_bar();                          // the rows and the gates may be restaged once every thread has read them
  }
}

// ================================================================================================= backward dz, dlogit
__global__ void __launch_bounds__(NTHREADS, 1)
ple_bwd_dz_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_rows, const __grid_constant__ Gates q,
                        const float* __restrict__ x, const float* __restrict__ be, const float* __restrict__ gates,
                        const float* __restrict__ g_out, float* __restrict__ dzbuf, int B, int d, int H, int DP, int HP,
                        int GP, int SB) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  const int ldx = DP + 4, ldp = q.GC + 1, nk = DP / KB, NJ = HP / PC, R = q.E * HP + GP;
  float* xs = reinterpret_cast<float*>(smem + SB * SBYTES);               // [64][ldx]   x rows
  float* dps = xs + TM * ldx;                                              // [64][ldp]   <g_o, h_e> (see dp_slot)
  const uint32_t sbase = smem_u32(smem);
  Ring ring(smem_u32(dps + TM * ldp), SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_tiles = (B + TM - 1) / TM;
  ring.init();
  // ============================ TMA producer: per expert, every 64 hidden units ============================
  if (producer_role(warp, lane, [&] {
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x)
          for (int e = 0; e < q.E; ++e)
            for (int j = 0; j < NJ; ++j)
              for (int kb = 0; kb < nk; ++kb) {
                const Ring::Slot slot = ring.acquire(SBYTES);
                load_stage(sbase + slot.stage * SBYTES, &tmap_rows, e * HP + j * PC, kb, R, slot.full);
              }
      }))
    return;

  // ============================ consumers ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3;
  const int r0 = w * 16 + g;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long base = (long long)tile * TM;
    const bool v0 = base + r0 < B, v1 = base + r0 + 8 < B;
    stage_tile(xs, ldx, x, base, B, d, DP);
    for (int idx = threadIdx.x; idx < TM * ldp; idx += NWG * 128) dps[idx] = 0.f;
    consumers_bar();
    float* dz0 = dzbuf + (size_t)(base + r0) * R;
    const float* p0 = gates + (size_t)(base + r0) * q.GC;
    for (int e = 0; e < q.E; ++e) {
      float pe[MAX_T][2], s[MAX_T][2];
#pragma unroll
      for (int o = 0; o < MAX_T; ++o) {
        pe[o][0] = o < q.O && v0 ? coef(q, p0, o, e) : 0.f;
        pe[o][1] = o < q.O && v1 ? coef(q, p0 + (size_t)8 * q.GC, o, e) : 0.f;
        s[o][0] = s[o][1] = 0.f;
      }
      for (int j = 0; j < NJ; ++j) {
        float a[HC / 2];
        gemm_ks(a, xs, ldx, nk, r0, t, lane, wg, ring, sbase);
        float gh[HC / 2];
#pragma unroll
        for (int k = 0; k < HC / 2; ++k) {    // h_e, and h_e > 0 exactly where a_e > 0
          const int col = j * PC + wg * HC + 8 * (k >> 2) + 2 * t + (k & 1);
          a[k] = fmaxf(a[k] + (col < H ? __ldg(be + (size_t)e * H + col) : 0.f), 0.f);
          gh[k] = 0.f;
        }
#pragma unroll
        for (int o = 0; o < MAX_T; ++o) {
          if (o >= q.O) break;
          const float* go = g_out + ((size_t)o * B + base + r0) * H;
#pragma unroll
          for (int k = 0; k < HC / 2; ++k) {
            const int col = j * PC + wg * HC + 8 * (k >> 2) + 2 * t + (k & 1);
            const bool hi = (k >> 1) & 1;
            const float gv = col < H && (hi ? v1 : v0) ? __ldg(go + (hi ? (size_t)8 * H : 0) + col) : 0.f;
            gh[k] = fmaf(pe[o][hi], gv, gh[k]);
            s[o][hi] = fmaf(gv, a[k], s[o][hi]);
          }
        }
#pragma unroll
        for (int c = 0; c < HC / 8; ++c) {
          const int col = e * HP + j * PC + wg * HC + 8 * c + 2 * t;
          const float2 lo = make_float2(a[4 * c] > 0.f ? gh[4 * c] : 0.f, a[4 * c + 1] > 0.f ? gh[4 * c + 1] : 0.f);
          const float2 hi = make_float2(a[4 * c + 2] > 0.f ? gh[4 * c + 2] : 0.f, a[4 * c + 3] > 0.f ? gh[4 * c + 3] : 0.f);
          if (v0) *reinterpret_cast<float2*>(dz0 + col) = lo;
          if (v1) *reinterpret_cast<float2*>(dz0 + (size_t)8 * R + col) = hi;
        }
      }
#pragma unroll
      for (int o = 0; o < MAX_T; ++o) {
        if (o >= q.O) break;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          s[o][r] += __shfl_xor_sync(0xffffffffu, s[o][r], 1);
          s[o][r] += __shfl_xor_sync(0xffffffffu, s[o][r], 2);
        }
        const int slot = dp_slot(q, o, e);
        if (t == 0 && slot >= 0) {            // the two warpgroups' halves: 0 + a + b is the same sum in either order
          atomicAdd(dps + r0 * ldp + slot, s[o][0]);
          atomicAdd(dps + (r0 + 8) * ldp + slot, s[o][1]);
        }
      }
    }
    consumers_bar();
    // softmax backward, one thread per (row, gate): dlogit_g[j] = p_g[j] (dp_g[j] - sum_j p_g[j] dp_g[j])
    for (int idx = threadIdx.x; idx < TM * (q.G + 1); idx += NWG * 128) {
      const int r = idx / (q.G + 1), gi = idx % (q.G + 1);
      if (base + r >= B) continue;
      float* dl = dzbuf + (size_t)(base + r) * R + q.E * HP;
      if (gi == q.G) {                        // the padding columns: zeros for the dx and dW GEMMs
        for (int c = q.GC; c < GP; ++c) dl[c] = 0.f;
        continue;
      }
      const float* p = gates + (size_t)(base + r) * q.GC + q.c0[gi];
      const float* dp = dps + r * ldp;
      const int len = gate_len(q, gi);
      float sum = 0.f;
      for (int j = 0; j < len; ++j) {
        const float dpj = dp[q.O == 1 ? gate_expert(q, gi, j) : q.c0[gi] + j];
        sum = fmaf(__ldg(p + j), dpj, sum);
      }
      for (int j = 0; j < len; ++j) {
        const float dpj = dp[q.O == 1 ? gate_expert(q, gi, j) : q.c0[gi] + j];
        dl[q.c0[gi] + j] = __ldg(p + j) * (dpj - sum);
      }
    }
    consumers_bar();                          // the rows and the dp table may be restaged once every thread is done
  }
}

// ================================================================================================= backward dx
__host__ __device__ constexpr int dx_stage_bytes(int N) { return DX_TILE * 128 + 2 * N * 128; }

// d_x[:, ds N ..] = [dz | dlogit] . [W | Gcat]^T over the R units: A = the workspace rows [128 samples x 32 units]
// (SWIZZLE_128B, read into registers), B = the hidden-layout operand [N inputs x 32 units] (hi | lo).
template <int N>
__global__ void __launch_bounds__(NTHREADS, 1)
ple_bwd_dx_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_dz, const __grid_constant__ CUtensorMap tmap_hidden,
                        float* __restrict__ d_x, int B, int d, int DH, int R, int n_ds, int SB) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int STB = dx_stage_bytes(N);
  const uint32_t sbase = smem_u32(smem);
  Ring ring(sbase + SB * STB, SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_work = (B + DX_TILE - 1) / DX_TILE * n_ds, nk = R / KB;
  ring.init();
  // ============================ TMA producer: per 32 units, the dz | dlogit rows and the operand ============================
  if (producer_role(warp, lane, [&] {
        for (int wk = blockIdx.x; wk < n_work; wk += gridDim.x) {
          const int tile = wk / n_ds, ds = wk % n_ds;
          for (int kb = 0; kb < nk; ++kb) {
            const Ring::Slot slot = ring.acquire(STB);
            const uint32_t dst = sbase + slot.stage * STB;
            tma_load_2d(dst, &tmap_dz, kb * KB, tile * DX_TILE, slot.full);
            tma_load_2d(dst + DX_TILE * 128, &tmap_hidden, kb * KB, ds * N, slot.full);
            tma_load_2d(dst + DX_TILE * 128 + N * 128, &tmap_hidden, kb * KB, DH + ds * N, slot.full);
          }
        }
      }))
    return;

  // ============================ consumers ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3;
  const int r0 = wg * WG_M + w * 16 + g;     // this thread's rows of the 128-sample tile: r0, r0 + 8
  for (int wk = blockIdx.x; wk < n_work; wk += gridDim.x) {
    const int tile = wk / n_ds, ds = wk % n_ds;
    float acc[N / 2], dacc[N / 2];
#pragma unroll
    for (int k = 0; k < N / 2; ++k) { acc[k] = 0.f; dacc[k] = 0.f; }
    for (int kb = 0; kb < nk; ++kb) {
      const uint32_t st = sbase + ring.wait() * STB;
      const float* as = reinterpret_cast<const float*>(smem + (st - sbase));
      uint32_t ah[4][4], al[4][4];
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        float a[4];
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) {    // element (row, k) of a SWIZZLE_128B tile: 16-byte chunk k / 4 XOR row % 8
          const int row = r0 + 8 * (qq & 1), k = 8 * ks + t + 4 * (qq >> 1);
          a[qq] = as[row * 32 + (((k >> 2) ^ (row & 7)) << 2) + (k & 3)];
        }
        tf32_split(a, ah[ks], al[ks]);
      }
      const uint64_t bhi = gmma_desc_kmajor(st + DX_TILE * 128, 128), blo = gmma_desc_kmajor(st + DX_TILE * 128 + N * 128, 128);
      const bool start = chain_first(kb, DX_KCHAIN);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) mma_3xtf32<N>(dacc, ah[ks], al[ks], bhi, blo, (uint64_t)(2 * ks), (start && ks == 0) ? 0 : 1);
      wgmma_commit();
      wgmma_wait_keep(ah, al);
      ring.release(lane);
      if (chain_last(kb, nk, DX_KCHAIN)) chain_drain(acc, dacc);
    }
    const long long row0 = (long long)tile * DX_TILE + r0;
#pragma unroll
    for (int c = 0; c < N / 8; ++c) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int k = ds * N + 8 * c + 2 * t + e;
        if (k < d) {
          if (row0 < B) d_x[(size_t)row0 * d + k] = acc[4 * c + e];
          if (row0 + 8 < B) d_x[(size_t)(row0 + 8) * d + k] = acc[4 * c + 2 + e];
        }
      }
    }
  }
}

// ================================================================================================= backward dW
__host__ __device__ constexpr int dw_smem_bytes(int N, int SB) { return SB * (2 * N * 128 + DW_BC * DW_NC * 4 + 16); }

// P = the workspace rows [dz_0 | .. | dz_{E-1} | dlogit] (B, R), Q = x[:, ds N ..]: row n < E HP of the result is
// dW_e[ds N .., h] (n = e HP + h) with db_e[h] its sum over the batch (added by the ds = 0 slice), row E HP + c is
// dGcat[ds N .., c].
template <int N>
__global__ void __launch_bounds__(NTHREADS, 1)
ple_bwd_dw_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_p, const float* __restrict__ x, float* __restrict__ d_we,
                        float* __restrict__ d_be, float* __restrict__ d_wg, int B, int d, int E, int H, int GC, int HP,
                        int ngroups, int nslices, int SB) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int qt_bytes = 2 * N * 128;                     // Q^T tiles [N x 32 samples] (hi | lo), 128B-swizzled
  constexpr int p_floats = DW_BC * DW_NC;                   // one P chunk [32 samples x 128 units]
  uint8_t* qts = smem;
  float* ps = reinterpret_cast<float*>(smem + SB * qt_bytes);
  Ring ring(smem_u32(ps + SB * p_floats), SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int group = blockIdx.x % ngroups, ds = blockIdx.y, k0 = ds * N;
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
  float acc[N / 2];
  batch_reduce<N>(
      acc, ring, qts, c_beg, c_end, B, lane, nl0, [](int) {},
      [&](int k, int b0, int b) { return k0 + k < d ? __ldg(x + (size_t)(b0 + b) * d + k0 + k) : 0.f; },
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
    } else if (n - E * HP < GC) {
      dst = d_wg + (n - E * HP);
      stride = GC;
    }
#pragma unroll
    for (int cc = 0; cc < N / 8; ++cc) {
#pragma unroll
      for (int xx = 0; xx < 2; ++xx) {
        const int k = k0 + 8 * cc + 2 * t + xx;
        if (dst != nullptr && k < d) atomicAdd(dst + (size_t)k * stride, acc[4 * cc + 2 * r + xx]);
      }
    }
    float v = rsum[r];
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    if (ds == 0 && t == 0 && n < E * HP && n % HP < H) atomicAdd(d_be + (size_t)(n / HP) * H + n % HP, v);
  }
}

}  // namespace ple
}  // namespace ctr

// ------------------------------------------------------------------------------------------------ host
using namespace ctr;
using namespace ctr::ple;

namespace {

struct PleShape {
  Gates q;
  int DP, DH, N;                   // x width padded to 32; hidden-operand rows (d padded to N); the dx / dW slice width
  int64_t HP, GP, R;
  int64_t rows_floats, hidden_floats;
  int64_t hidden_offset, dz_offset; // workspace byte offsets of the hidden operand and of the dz | dlogit rows (B, R)
  int64_t fwd_bytes, bwd_bytes;
};

// Checks the sizes and fills the gate structure; `fn` names the entry in the messages.
int shape_of(const char* fn, int64_t B, int64_t d, int64_t H, int64_t T, const int64_t* experts_per_task, int64_t S,
             int64_t extraction, PleShape& s) {
  CTR_REQUIRE(experts_per_task != nullptr, "%s: null argument (experts_per_task)", fn);
  CTR_REQUIRE(B >= 0 && d >= 1 && H >= 1 && T >= 1 && S >= 1 && (extraction == 0 || extraction == 1),
              "%s: bad sizes B=%lld d=%lld H=%lld T=%lld S=%lld extraction=%lld", fn, (long long)B, (long long)d,
              (long long)H, (long long)T, (long long)S, (long long)extraction);
  CTR_UNSUPPORTED(d > MAX_D, "%s: unsupported input width d=%lld (the tensor-core kernels take d <= %d)", fn, (long long)d,
                  MAX_D);
  CTR_UNSUPPORTED(H > MAX_H, "%s: unsupported expert_hidden_units H=%lld (the tensor-core kernels take H <= %d)", fn,
                  (long long)H, MAX_H);
  CTR_UNSUPPORTED(T > MAX_T, "%s: unsupported number of tasks T=%lld (the tensor-core kernels take T <= %d)", fn,
                  (long long)T, MAX_T);
  int64_t sum_n = 0;
  for (int64_t t = 0; t < T; ++t) {
    CTR_REQUIRE(experts_per_task[t] >= 1, "%s: bad experts_per_task[%lld]=%lld (at least 1)", fn, (long long)t,
                (long long)experts_per_task[t]);
    CTR_UNSUPPORTED(experts_per_task[t] > MAX_E, "%s: unsupported experts_per_task[%lld]=%lld (E <= %d)", fn, (long long)t,
                    (long long)experts_per_task[t], MAX_E);
    sum_n += experts_per_task[t];
  }
  CTR_UNSUPPORTED(S > MAX_E, "%s: unsupported num_experts_in_shared S=%lld (E <= %d)", fn, (long long)S, MAX_E);
  const int64_t E = sum_n + S, GC = sum_n + T * S + (extraction ? E : 0);
  CTR_UNSUPPORTED(E > MAX_E, "%s: unsupported expert count E=%lld (the tensor-core kernels take E <= %d)", fn, (long long)E,
                  MAX_E);
  CTR_UNSUPPORTED(GC > MAX_GC, "%s: unsupported gate width GC=%lld (the tensor-core kernels take GC <= %d)", fn,
                  (long long)GC, MAX_GC);
  CTR_UNSUPPORTED(B > 0x7fffff00LL, "%s: batch too large (B=%lld)", fn, (long long)B);
  Gates& q = s.q;
  q.T = (int)T; q.S = (int)S; q.E = (int)E; q.ES = (int)sum_n; q.G = (int)(T + extraction); q.O = extraction ? 1 : (int)T;
  q.GC = (int)GC;
  int e0 = 0, c0 = 0;
  for (int t = 0; t < MAX_T; ++t) {
    q.n[t] = t < T ? (int)experts_per_task[t] : 0;
    q.e0[t] = e0;
    e0 += q.n[t];
  }
  for (int g = 0; g <= MAX_T; ++g) {
    q.c0[g] = c0;
    if (g < q.G) c0 += gate_len(q, g);
  }
  s.DP = (int)pad_to(d, KB);
  s.N = d <= 32 ? 32 : d <= 64 ? 64 : 128;
  s.DH = (int)pad_to(d, s.N);
  s.HP = pad_to(H, PC);
  s.GP = pad_to(GC, PC);
  s.R = E * s.HP + s.GP;
  s.rows_floats = 2 * s.R * s.DP;
  s.hidden_floats = 2 * s.R * s.DH;
  s.fwd_bytes = pad_to(s.rows_floats * 4, 128);
  s.hidden_offset = s.fwd_bytes;
  s.dz_offset = s.hidden_offset + pad_to(s.hidden_floats * 4, 128);
  s.bwd_bytes = s.dz_offset + pad_to(B * s.R * 4, 128);
  return CTR_OK;
}

// ring stages of the forward / dz kernels next to their x tile and gate table: as many as fit, at most 4
int tile_stages(const PleShape& s) {
  int sb = 4;
  while (sb > 2 && tile_bytes(s.DP, s.q.GC, sb) + 1024 > (int)SMEM_CAP) --sb;
  return sb;
}
static_assert(tile_bytes(MAX_D, MAX_GC, 2) + 1024 <= (int)SMEM_CAP, "forward / dz shared memory at the bounds");

int prep(const char* what, const float* we, const float* wg, void* ws, int64_t d, int64_t H, const PleShape& s, int nslots,
         cudaStream_t st) {
  float* rows = static_cast<float*>(ws);
  float* hidden = reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + s.hidden_offset);
  return launch(what, ple_prep_kernel, dim3(capped_grid((s.R * std::max(s.DP, s.DH) + 255) / 256, 1024), nslots), 256, 0,
                st, we, wg, rows, hidden, (int)d, s.q.E, (int)H, s.q.GC, s.DP, s.DH, (int)s.HP, (int)s.R);
}

}  // namespace

extern "C" int ctr_ple_workspace_bytes(int64_t B, int64_t d, int64_t H, int64_t T, const int64_t* experts_per_task,
                                       int64_t S, int64_t extraction, int64_t* bytes) {
  static const char* fn = "ctr_ple_workspace_bytes";
  PleShape s;
  int rc = shape_of(fn, B, d, H, T, experts_per_task, S, extraction, s);
  if (rc) return rc;
  CTR_REQUIRE(bytes != nullptr, "ctr_ple_workspace_bytes: null argument");
  *bytes = s.bwd_bytes;
  return CTR_OK;
}

extern "C" int ctr_ple_fwd(const float* x, const float* w_experts, const float* b_experts, const float* w_gates, int64_t B,
                           int64_t d, int64_t H, int64_t T, const int64_t* experts_per_task, int64_t S, int64_t extraction,
                           float* out, float* gates, void* workspace, int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_ple_fwd";
  PleShape s;
  int rc = shape_of(fn, B, d, H, T, experts_per_task, S, extraction, s);
  if (rc) return rc;
  CTR_REQUIRE(x && w_experts && b_experts && w_gates && out && gates, "ctr_ple_fwd: null argument");
  rc = check_workspace(fn, "ctr_ple_workspace_bytes with B = 0", workspace, workspace_bytes, s.fwd_bytes);
  if (rc) return rc;
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  if ((rc = prep("ctr_ple_fwd(prep)", w_experts, w_gates, workspace, d, H, s, 1, st))) return rc;
  CUtensorMap mr;
  if ((rc = encode_2d(fn, &mr, workspace, s.DP, 2 * s.R, KB, PC, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  // Small batches split the hidden units of each tile over several CTAs (each recomputes the tile's gates) to fill the SMs.
  const int sms = sm_count();
  const int64_t n_tiles = (B + TM - 1) / TM;
  const int nsplit = (int)std::max<int64_t>(1, std::min<int64_t>(sms / n_tiles, s.HP / PC));
  const int sb = tile_stages(s);
  return launch("ctr_ple_fwd(wgmma)", ple_fwd_wgmma_kernel, capped_grid(n_tiles * nsplit, sms), NTHREADS,
                tile_bytes(s.DP, s.q.GC, sb) + 1024, st, mr, s.q, x, b_experts, out, gates, (int)B, (int)d, (int)H, s.DP,
                (int)s.HP, (int)s.GP, nsplit, sb);
}

extern "C" int ctr_ple_bwd(const float* x, const float* w_experts, const float* b_experts, const float* w_gates,
                           const float* gates, const float* g_out, int64_t B, int64_t d, int64_t H, int64_t T,
                           const int64_t* experts_per_task, int64_t S, int64_t extraction, float* d_x, float* d_w_experts,
                           float* d_b_experts, float* d_w_gates, void* workspace, int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_ple_bwd";
  PleShape s;
  int rc = shape_of(fn, B, d, H, T, experts_per_task, S, extraction, s);
  if (rc) return rc;
  CTR_REQUIRE(x && w_experts && b_experts && w_gates && gates && g_out && d_x && d_w_experts && d_b_experts && d_w_gates,
              "ctr_ple_bwd: null argument");
  rc = check_workspace(fn, "ctr_ple_workspace_bytes", workspace, workspace_bytes, s.bwd_bytes);
  if (rc) return rc;
  cudaStream_t st = as_stream(stream);
  const int64_t E = s.q.E;
  CTR_CUDA(cudaMemsetAsync(d_w_experts, 0, sizeof(float) * (size_t)(E * d * H), st));
  CTR_CUDA(cudaMemsetAsync(d_b_experts, 0, sizeof(float) * (size_t)(E * H), st));
  CTR_CUDA(cudaMemsetAsync(d_w_gates, 0, sizeof(float) * (size_t)(d * s.q.GC), st));
  if (B == 0) return CTR_OK;
  float* dzbuf = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + s.dz_offset);
  if ((rc = prep("ctr_ple_bwd(prep)", w_experts, w_gates, workspace, d, H, s, 2, st))) return rc;
  CUtensorMap mr, mh, mdx, mdw;
  if ((rc = encode_2d(fn, &mr, workspace, s.DP, 2 * s.R, KB, PC, CU_TENSOR_MAP_SWIZZLE_128B)) ||
      (rc = encode_2d(fn, &mh, static_cast<uint8_t*>(workspace) + s.hidden_offset, s.R, 2 * s.DH, KB, s.N,
                      CU_TENSOR_MAP_SWIZZLE_128B)) ||
      (rc = encode_2d(fn, &mdx, dzbuf, s.R, B, KB, DX_TILE, CU_TENSOR_MAP_SWIZZLE_128B)) ||
      (rc = encode_2d(fn, &mdw, dzbuf, s.R, B, DW_NC, DW_BC, CU_TENSOR_MAP_SWIZZLE_NONE)))
    return rc;
  const int sms = sm_count();
  const int sb = tile_stages(s);
  if ((rc = launch("ctr_ple_bwd(dz, wgmma)", ple_bwd_dz_wgmma_kernel, capped_grid((B + TM - 1) / TM, sms), NTHREADS,
                   tile_bytes(s.DP, s.q.GC, sb) + 1024, st, mr, s.q, x, b_experts, gates, g_out, dzbuf, (int)B, (int)d,
                   (int)H, s.DP, (int)s.HP, (int)s.GP, sb)))
    return rc;
  const int n_ds = s.DH / s.N;
  const int64_t n_dx = (B + DX_TILE - 1) / DX_TILE * n_ds;
  const int ngroups = (int)((s.R + DW_NC - 1) / DW_NC);
  const int nslices = batch_slices(sms / n_ds > 0 ? sms / n_ds : 1, ngroups, (B + DW_BC - 1) / DW_BC);
  return with_const<32, 64, 128>(s.N, [&](auto N) {
    constexpr int dx_sb = (int)((SMEM_CAP - 1024) / dx_stage_bytes(N)) < 4 ? (int)((SMEM_CAP - 1024) / dx_stage_bytes(N)) : 4;
    static_assert(dx_sb * (dx_stage_bytes(N) + 16) + 1024 <= (int)SMEM_CAP, "dx shared memory");
    if (int r = launch("ctr_ple_bwd(dx, wgmma)", ple_bwd_dx_wgmma_kernel<N>, capped_grid(n_dx, sms), NTHREADS,
                       dx_sb * (dx_stage_bytes(N) + 16) + 1024, st, mdx, mh, d_x, (int)B, (int)d, s.DH, (int)s.R, n_ds,
                       dx_sb))
      return r;
    const int dw_sb = stages_that_fit(1024, dw_smem_bytes(N, 1));
    return launch("ctr_ple_bwd(dw, wgmma)", ple_bwd_dw_wgmma_kernel<N>, dim3(ngroups * nslices, n_ds), NTHREADS,
                  dw_smem_bytes(N, dw_sb) + 1024, st, mdw, x, d_w_experts, d_b_experts, d_w_gates, (int)B, (int)d, s.q.E,
                  (int)H, s.q.GC, (int)s.HP, ngroups, nslices, dw_sb);
  });
}

// DeepCrossing residual unit -- DeepCrossing/residual_unit.py:4-21, applied in a loop at DeepCrossing/deepcrossing.py:149-153.
//
//   a   = x . W0 + b0     (B,H)      W0 = dense_{index}_0/kernel (d,H),  b0 (H)
//   h   = relu(a)
//   y   = h . W1 + b1     (B,d)      W1 = dense_{index}_1/kernel (H,d),  b1 (d)
//   out = relu(x + y)
// Backward, g = dL/dout:  gy = g [out > 0],  gh = (gy . W1^T) [a > 0],  dx = gy + gh . W0^T,
//                         dW1 = h^T . gy,  db1 = sum_b gy,  dW0 = x^T . gh,  db0 = sum_b gh.
//
// H100 mapping (the CIN / PNN pipeline of csrc/tc_ptx.cuh): two consumer warpgroups of 64 samples + one TMA producer warp,
// wgmma m64nNk8 kind tf32 with A in registers, 3xTF32 split for fp32-class accuracy, hidden-sized sums drained every 96
// chained MMAs.  The weights are prepped once per call into the caller's workspace as tf32 hi | lo copies, zero padded to
// DP = d rounded up to 32 / 64 / 96 / 128 and HP = H rounded up to HC = 32, in the K-major layouts the TMA tiles stream.
//   resunit_fwd_wgmma_kernel     per hidden chunk of HC units: a = x . W0[:, chunk] (A = x rows staged in shared memory,
//                                B = W0^T chunk), h = relu(a + b0) in registers, y += h . W1[chunk, :] (B = W1^T chunk).
//                                Epilogue relu(x + y + b1).  h never leaves the registers of the thread that computed it.
//   resunit_bwd_dx_wgmma_kernel  per chunk: a recomputed as in the forward, t = gy . W1^T[:, chunk] (B = W1 chunk),
//                                gh = t [a > 0], dx += gh . W0[chunk]^T (B = W0 chunk).  Writes h and gh (B, HP) to the
//                                workspace for the weight gradients; sums gy over its rows for db1.
//   resunit_bwd_dw_wgmma_kernel  dW1 = h^T . gy and dW0^T = gh^T . x, with sum_b gh = db0 alongside: A = h^T or gh^T (rows =
//                                hidden units, K = samples) from TMA-staged [32 samples x 128 units] chunks, B = gy^T or x^T
//                                [DP x 32 samples] generated on chip into 128B-swizzled shared memory.  A CTA owns 128 hidden
//                                units and a batch slice, and issues one atomic add per element at the end.  The
//                                consumer loop is tc_ptx.cuh's batch_reduce, shared with the PNN weight gradients.
// The rows of x, out and g are d floats (328 B at the reference d = 82), not a multiple of 16 bytes, so they are staged with
// ordinary loads; only the prepped weights and the workspace's h / gh (pitch HP) are TMA tensors.
//
// h feeds the second GEMM straight from the accumulator registers of the first: the prep kernel permutes the hidden rows of
// W1 (and of W0 for the backward's gh . W0^T) within each group of 8 to match the accumulator's column order (perm8 and the
// row-chunk GEMMs live in tc_ptx.cuh, shared with csrc/mmoe.cu).  The alternative, a round trip of h through shared memory,
// would cost a store, a warpgroup barrier and a load per chunk for nothing.
//
// Tensor path (the only path): d <= 128, 1 <= H <= 1024, any B >= 0.  Other shapes return CTR_ERR_UNSUPPORTED.
#include "tc_ptx.cuh"

namespace ctr {
namespace resunit {
using namespace ctr::tc;
using namespace ctr::tc::rows;

constexpr int TILE = NWG * WG_M;             // samples per CTA tile (forward, dx)

// Writes the tf32 hi | lo copies of the weights, zero padded, one layout per blockIdx.y slot (2 HP DP floats each):
//   0: W0^T [HP][DP]    1: W1^T [DP][HP] hidden order perm8    2: W1 [HP][DP]    3: W0 [DP][HP] hidden order perm8
__global__ void resunit_prep_kernel(const float* __restrict__ w0, const float* __restrict__ w1, float* __restrict__ dst,
                                    int d, int H, int DP, int HP, int4 layouts) {
  const int slot = blockIdx.y;
  const int L = slot == 0 ? layouts.x : slot == 1 ? layouts.y : layouts.z;
  const size_t total = (size_t)HP * DP;
  float* o = dst + 2 * total * slot;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    int i, j;
    if (L == 0 || L == 2) { j = (int)(idx / DP); i = (int)(idx % DP); }
    else { i = (int)(idx / HP); j = perm8((int)(idx % HP)); }
    float v = 0.f;
    if (i < d && j < H) v = (L == 0 || L == 3) ? __ldg(w0 + (size_t)i * H + j) : __ldg(w1 + (size_t)j * d + i);
    store_split(o, total, idx, v);
  }
}

// ================================================================================================= forward
__host__ __device__ constexpr int fwd_smem_bytes(int DP, int SB) {
  return SB * stage_bytes(DP) + NWG * WG_M * row_pitch(DP) * 4 + 16 * SB;
}

template <int DP, int SB>
__global__ void __launch_bounds__(NTHREADS, 1)
resunit_fwd_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_w0t, const __grid_constant__ CUtensorMap tmap_w1t,
                         const float* __restrict__ x, const float* __restrict__ b0, const float* __restrict__ b1,
                         float* __restrict__ out, int B, int d, int H, int HP) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int SBYTES = stage_bytes(DP), LD = row_pitch(DP);
  float* xs = reinterpret_cast<float*>(smem + SB * SBYTES);               // [2][64][LD]
  const uint32_t sbase = smem_u32(smem);
  Ring ring(smem_u32(xs + NWG * WG_M * LD), SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_tiles = (B + TILE - 1) / TILE, NC = HP / HC;
  ring.init();
  // ============================ TMA producer: per chunk, W0^T then W1^T (hi, lo) ============================
  if (producer_role(warp, lane, [&] {
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
          for (int j = 0; j < NC; ++j) {
            Ring::Slot slot = ring.acquire(SBYTES);
            load_rows_operand<DP>(sbase + slot.stage * SBYTES, &tmap_w0t, j, HP, slot.full);
            slot = ring.acquire(SBYTES);
            load_hidden_operand<DP>(sbase + slot.stage * SBYTES, &tmap_w1t, j, slot.full);
          }
        }
      }))
    return;

  // ============================ consumers ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3, tw = threadIdx.x & 127;
  const int r0 = w * 16 + g;
  float* xw = xs + wg * WG_M * LD;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long base = (long long)tile * TILE + wg * WG_M;
    stage_rows<DP>(xw, x, nullptr, base, B, d, tw);
    wg_bar_sync(1 + wg);
    float acc[DP / 2], dacc[DP / 2];
#pragma unroll
    for (int q = 0; q < DP / 2; ++q) { acc[q] = 0.f; dacc[q] = 0.f; }
    for (int j = 0; j < NC; ++j) {
      float a[HC / 2];
      gemm_rows<DP>(a, xw, r0, t, sbase + ring.wait() * SBYTES);
      ring.release(lane);
#pragma unroll
      for (int c = 0; c < HC / 8; ++c) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = j * HC + 8 * c + 2 * t + e;
          const float bv = col < H ? __ldg(b0 + col) : 0.f;
          a[4 * c + e] = fmaxf(a[4 * c + e] + bv, 0.f);
          a[4 * c + 2 + e] = fmaxf(a[4 * c + 2 + e] + bv, 0.f);
        }
      }
      uint32_t hh[HC / 8][4], hl[HC / 8][4];
      acc_to_a(a, hh, hl);
      gemm_hidden<DP>(dacc, hh, hl, sbase + ring.wait() * SBYTES, chain_first(j, CHAIN));
      ring.release(lane);
      if (chain_last(j, NC, CHAIN)) chain_drain(acc, dacc);
    }
#pragma unroll
    for (int c = 0; c < DP / 8; ++c) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int i = 8 * c + 2 * t + e;
        if (i < d) {
          const float bv = __ldg(b1 + i);
          if (base + r0 < B) out[(size_t)(base + r0) * d + i] = fmaxf(xw[r0 * LD + i] + (acc[4 * c + e] + bv), 0.f);
          if (base + r0 + 8 < B)
            out[(size_t)(base + r0 + 8) * d + i] = fmaxf(xw[(r0 + 8) * LD + i] + (acc[4 * c + 2 + e] + bv), 0.f);
        }
      }
    }
    wg_bar_sync(1 + wg);                      // the rows may be restaged once every thread has read them
  }
}

// ================================================================================================= backward dx
__host__ __device__ constexpr int dx_smem_bytes(int DP, int SB) {
  return SB * stage_bytes(DP) + 2 * NWG * WG_M * row_pitch(DP) * 4 + 16 * SB;
}

template <int DP, int SB>
__global__ void __launch_bounds__(NTHREADS, 1)
resunit_bwd_dx_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_w0t, const __grid_constant__ CUtensorMap tmap_w1,
                            const __grid_constant__ CUtensorMap tmap_w0p, const float* __restrict__ x,
                            const float* __restrict__ b0, const float* __restrict__ outv, const float* __restrict__ g_out,
                            float* __restrict__ d_x, float* __restrict__ hbuf, float* __restrict__ ghbuf,
                            float* __restrict__ d_b1, int B, int d, int H, int HP) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  constexpr int SBYTES = stage_bytes(DP), LD = row_pitch(DP);
  float* xs = reinterpret_cast<float*>(smem + SB * SBYTES);               // [2][64][LD]  x rows
  float* gs = xs + NWG * WG_M * LD;                                        // [2][64][LD]  gy rows
  const uint32_t sbase = smem_u32(smem);
  Ring ring(smem_u32(gs + NWG * WG_M * LD), SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_tiles = (B + TILE - 1) / TILE, NC = HP / HC;
  ring.init();
  // ============================ TMA producer: per chunk, W0^T, W1 and W0 (hi, lo) ============================
  if (producer_role(warp, lane, [&] {
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
          for (int j = 0; j < NC; ++j) {
            Ring::Slot slot = ring.acquire(SBYTES);
            load_rows_operand<DP>(sbase + slot.stage * SBYTES, &tmap_w0t, j, HP, slot.full);
            slot = ring.acquire(SBYTES);
            load_rows_operand<DP>(sbase + slot.stage * SBYTES, &tmap_w1, j, HP, slot.full);
            slot = ring.acquire(SBYTES);
            load_hidden_operand<DP>(sbase + slot.stage * SBYTES, &tmap_w0p, j, slot.full);
          }
        }
      }))
    return;

  // ============================ consumers ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3, tw = threadIdx.x & 127;
  const int r0 = w * 16 + g;
  float* xw = xs + wg * WG_M * LD;
  float* gw = gs + wg * WG_M * LD;
  float db1 = 0.f;                            // column tw of gy, summed over this warpgroup's rows
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long base = (long long)tile * TILE + wg * WG_M;
    stage_rows<DP>(xw, x, nullptr, base, B, d, tw);
    stage_rows<DP>(gw, g_out, outv, base, B, d, tw);
    wg_bar_sync(1 + wg);
    if (tw < d)
      for (int r = 0; r < WG_M; ++r) db1 += gw[r * LD + tw];
    const bool v0 = base + r0 < B, v1 = base + r0 + 8 < B;
    float* h0 = hbuf + (size_t)(base + r0) * HP;
    float* gh0 = ghbuf + (size_t)(base + r0) * HP;
    float acc[DP / 2], dacc[DP / 2];
#pragma unroll
    for (int q = 0; q < DP / 2; ++q) { acc[q] = 0.f; dacc[q] = 0.f; }
    for (int j = 0; j < NC; ++j) {
      float a[HC / 2];
      gemm_rows<DP>(a, xw, r0, t, sbase + ring.wait() * SBYTES);
      ring.release(lane);
      uint32_t live = 0;                      // bit q: a[q] + b0 > 0
#pragma unroll
      for (int c = 0; c < HC / 8; ++c) {
        const int col = j * HC + 8 * c + 2 * t;
        const float bv0 = col < H ? __ldg(b0 + col) : 0.f, bv1 = col + 1 < H ? __ldg(b0 + col + 1) : 0.f;
        const float p[4] = {a[4 * c] + bv0, a[4 * c + 1] + bv1, a[4 * c + 2] + bv0, a[4 * c + 3] + bv1};
#pragma unroll
        for (int e = 0; e < 4; ++e) live |= (p[e] > 0.f ? 1u : 0u) << (4 * c + e);
        if (v0) *reinterpret_cast<float2*>(h0 + col) = make_float2(fmaxf(p[0], 0.f), fmaxf(p[1], 0.f));
        if (v1) *reinterpret_cast<float2*>(h0 + (size_t)8 * HP + col) = make_float2(fmaxf(p[2], 0.f), fmaxf(p[3], 0.f));
      }
      float gh[HC / 2];
      gemm_rows<DP>(gh, gw, r0, t, sbase + ring.wait() * SBYTES);
      ring.release(lane);
#pragma unroll
      for (int q = 0; q < HC / 2; ++q) gh[q] = (live >> q) & 1u ? gh[q] : 0.f;
#pragma unroll
      for (int c = 0; c < HC / 8; ++c) {
        const int col = j * HC + 8 * c + 2 * t;
        if (v0) *reinterpret_cast<float2*>(gh0 + col) = make_float2(gh[4 * c], gh[4 * c + 1]);
        if (v1) *reinterpret_cast<float2*>(gh0 + (size_t)8 * HP + col) = make_float2(gh[4 * c + 2], gh[4 * c + 3]);
      }
      uint32_t hh[HC / 8][4], hl[HC / 8][4];
      acc_to_a(gh, hh, hl);
      gemm_hidden<DP>(dacc, hh, hl, sbase + ring.wait() * SBYTES, chain_first(j, CHAIN));
      ring.release(lane);
      if (chain_last(j, NC, CHAIN)) chain_drain(acc, dacc);
    }
#pragma unroll
    for (int c = 0; c < DP / 8; ++c) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int i = 8 * c + 2 * t + e;
        if (i < d) {
          if (v0) d_x[(size_t)(base + r0) * d + i] = gw[r0 * LD + i] + acc[4 * c + e];
          if (v1) d_x[(size_t)(base + r0 + 8) * d + i] = gw[(r0 + 8) * LD + i] + acc[4 * c + 2 + e];
        }
      }
    }
    wg_bar_sync(1 + wg);
  }
  if (tw < d) atomicAdd(d_b1 + tw, db1);
}

// ================================================================================================= backward dW
__host__ __device__ constexpr int dw_smem_bytes(int DP, int SB) { return SB * (2 * DP * 128 + DW_BC * DW_NC * 4 + 16); }

// MODE 0: P = h, Q = gy = g [out > 0]: dw = dW1 (H,d).   MODE 1: P = gh, Q = x: dw = dW0 (d,H), db = db0 (H).
template <int DP, int MODE>
__global__ void __launch_bounds__(NTHREADS, 1)
resunit_bwd_dw_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_p, const float* __restrict__ q,
                            const float* __restrict__ qmask, float* __restrict__ dw, float* __restrict__ db, int B, int d,
                            int H, int ngroups, int nslices, int SB) {
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

  // ============================ consumers: B = Q^T generated from q, A = P^T ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3;
  float rsum[2] = {0.f, 0.f};                               // MODE 1: sum_b gh of this thread's two units
  const int nl0 = wg * WG_M + w * 16 + g;                   // this thread's A rows: units n0 + nl0 (+8)
  float acc[DP / 2];
  batch_reduce<DP>(
      acc, ring, qts, c_beg, c_end, B, lane, nl0, [](int) {},
      [&](int k, int b0, int b) {
        if (k >= d) return 0.f;
        const size_t o = (size_t)(b0 + b) * d + k;
        return (MODE == 1 || __ldg(qmask + o) > 0.f) ? __ldg(q + o) : 0.f;
      },
      [&](int s, int b, int nl) {
        const float v = ps[(size_t)s * p_floats + b * DW_NC + nl];
        if (MODE == 1) rsum[nl == nl0 ? 0 : 1] += v;
        return v;
      });
  if (c_end <= c_beg) return;
#pragma unroll
  for (int cc = 0; cc < DP / 8; ++cc) {
#pragma unroll
    for (int x = 0; x < 2; ++x) {
      const int i = 8 * cc + 2 * t + x;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int j = n0 + nl0 + 8 * r;
        if (i < d && j < H) atomicAdd(MODE == 0 ? dw + (size_t)j * d + i : dw + (size_t)i * H + j, acc[4 * cc + 2 * r + x]);
      }
    }
  }
  if (MODE == 1) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float v = rsum[r];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      const int j = n0 + nl0 + 8 * r;
      if (t == 0 && j < H) atomicAdd(db + j, v);
    }
  }
}

}  // namespace resunit
}  // namespace ctr

// ------------------------------------------------------------------------------------------------ host
using namespace ctr;
using namespace ctr::resunit;

namespace {

struct RuShape {
  int DP;
  int64_t HP;
  int64_t slot_floats;             // one prepped layout: hi | lo copies of [HP][DP] or [DP][HP]
  int64_t h_offset, gh_offset;     // workspace byte offsets of h and gh (B, HP) (backward)
  int64_t fwd_bytes, bwd_bytes;
};

RuShape shape_of(int64_t B, int64_t d, int64_t H) {
  RuShape s;
  s.DP = dp_class(d);
  s.HP = pad_to(H, HC);
  s.slot_floats = 2 * s.HP * s.DP;
  s.fwd_bytes = pad_to(2 * s.slot_floats * (int64_t)sizeof(float), 128);
  s.h_offset = pad_to(3 * s.slot_floats * (int64_t)sizeof(float), 128);
  s.gh_offset = s.h_offset + pad_to(B * s.HP * (int64_t)sizeof(float), 128);
  s.bwd_bytes = s.gh_offset + pad_to(B * s.HP * (int64_t)sizeof(float), 128);
  return s;
}

int check_shape(const char* fn, int64_t B, int64_t d, int64_t H) {
  CTR_REQUIRE(B >= 0 && d >= 1 && H >= 1, "%s: bad sizes B=%lld d=%lld H=%lld", fn, (long long)B, (long long)d, (long long)H);
  CTR_UNSUPPORTED(d > 128, "%s: unsupported input width d=%lld (the tensor-core kernels take d <= 128)", fn, (long long)d);
  CTR_UNSUPPORTED(H > 1024, "%s: unsupported internal_dim H=%lld (the tensor-core kernels take H <= 1024)", fn, (long long)H);
  CTR_UNSUPPORTED(B > 0x7fffff00LL, "%s: batch too large (B=%lld)", fn, (long long)B);
  return CTR_OK;
}

// prepped layout in workspace slot `slot`, as a rows operand ([2 HP][DP], boxes of [HC x 32]) or a hidden operand
// ([2 DP][HP], boxes of [DP x 32])
int encode_weights(const char* fn, CUtensorMap* map, float* ws, const RuShape& s, int slot, bool rows) {
  const float* base = ws + s.slot_floats * slot;
  return rows ? encode_rows_operand(fn, map, base, s.DP, s.HP) : encode_hidden_operand(fn, map, base, s.DP, s.HP);
}

int prep(const char* what, const float* w0, const float* w1, float* ws, int64_t d, int64_t H, const RuShape& s, int nslots,
         int4 layouts, cudaStream_t st) {
  return launch(what, resunit_prep_kernel, dim3(capped_grid((s.HP * s.DP + 255) / 256, 1024), nslots), 256, 0, st, w0, w1,
                ws, (int)d, (int)H, s.DP, (int)s.HP, layouts);
}

}  // namespace

extern "C" int ctr_residual_unit_workspace_bytes(int64_t B, int64_t d, int64_t H, int64_t* bytes) {
  int rc = check_shape("ctr_residual_unit_workspace_bytes", B, d, H);
  if (rc) return rc;
  CTR_REQUIRE(bytes != nullptr, "ctr_residual_unit_workspace_bytes: null argument");
  *bytes = shape_of(B, d, H).bwd_bytes;
  return CTR_OK;
}

extern "C" int ctr_residual_unit_fwd(const float* x, const float* w0, const float* b0, const float* w1, const float* b1,
                                     int64_t B, int64_t d, int64_t H, float* out, void* workspace, int64_t workspace_bytes,
                                     void* stream) {
  static const char* fn = "ctr_residual_unit_fwd";
  int rc = check_shape(fn, B, d, H);
  if (rc) return rc;
  CTR_REQUIRE(x && w0 && b0 && w1 && b1 && out, "ctr_residual_unit_fwd: null argument");
  const RuShape s = shape_of(B, d, H);
  rc = check_workspace(fn, "ctr_residual_unit_workspace_bytes with B = 0", workspace, workspace_bytes, s.fwd_bytes);
  if (rc) return rc;
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  float* ws = static_cast<float*>(workspace);
  rc = prep("ctr_residual_unit_fwd(prep)", w0, w1, ws, d, H, s, 2, make_int4(0, 1, -1, 0), st);
  if (rc) return rc;
  CUtensorMap m0, m1;
  if ((rc = encode_weights(fn, &m0, ws, s, 0, true)) || (rc = encode_weights(fn, &m1, ws, s, 1, false))) return rc;
  const int grid = capped_grid((B + TILE - 1) / TILE, sm_count());
  return with_const<32, 64, 96, 128>(s.DP, [&](auto DP) {
    constexpr int SB = 4;
    static_assert(fwd_smem_bytes(DP, SB) + 1024 <= SMEM_CAP, "forward shared memory");
    return launch("ctr_residual_unit_fwd(wgmma)", resunit_fwd_wgmma_kernel<DP, SB>, grid, NTHREADS,
                  fwd_smem_bytes(DP, SB) + 1024, st, m0, m1, x, b0, b1, out, (int)B, (int)d, (int)H, (int)s.HP);
  });
}

extern "C" int ctr_residual_unit_bwd(const float* x, const float* w0, const float* b0, const float* w1, const float* b1,
                                     const float* out, const float* g_out, int64_t B, int64_t d, int64_t H, float* d_x,
                                     float* d_w0, float* d_b0, float* d_w1, float* d_b1, void* workspace,
                                     int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_residual_unit_bwd";
  int rc = check_shape(fn, B, d, H);
  if (rc) return rc;
  CTR_REQUIRE(x && w0 && b0 && w1 && b1 && out && g_out && d_x && d_w0 && d_b0 && d_w1 && d_b1,
              "ctr_residual_unit_bwd: null argument");
  const RuShape s = shape_of(B, d, H);
  rc = check_workspace(fn, "ctr_residual_unit_workspace_bytes", workspace, workspace_bytes, s.bwd_bytes);
  if (rc) return rc;
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(d_w0, 0, sizeof(float) * (size_t)(d * H), st));
  CTR_CUDA(cudaMemsetAsync(d_w1, 0, sizeof(float) * (size_t)(d * H), st));
  CTR_CUDA(cudaMemsetAsync(d_b0, 0, sizeof(float) * (size_t)H, st));
  CTR_CUDA(cudaMemsetAsync(d_b1, 0, sizeof(float) * (size_t)d, st));
  if (B == 0) return CTR_OK;
  float* ws = static_cast<float*>(workspace);
  float* hbuf = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + s.h_offset);
  float* ghbuf = reinterpret_cast<float*>(static_cast<uint8_t*>(workspace) + s.gh_offset);
  rc = prep("ctr_residual_unit_bwd(prep)", w0, w1, ws, d, H, s, 3, make_int4(0, 2, 3, 0), st);
  if (rc) return rc;
  CUtensorMap m0, m2, m3, mh, mgh;
  if ((rc = encode_weights(fn, &m0, ws, s, 0, true)) || (rc = encode_weights(fn, &m2, ws, s, 1, true)) ||
      (rc = encode_weights(fn, &m3, ws, s, 2, false)) ||
      (rc = encode_2d(fn, &mh, hbuf, s.HP, B, DW_NC, DW_BC, CU_TENSOR_MAP_SWIZZLE_NONE)) ||
      (rc = encode_2d(fn, &mgh, ghbuf, s.HP, B, DW_NC, DW_BC, CU_TENSOR_MAP_SWIZZLE_NONE)))
    return rc;
  const int sms = sm_count();
  const int grid = capped_grid((B + TILE - 1) / TILE, sms);
  const int ngroups = (int)((s.HP + DW_NC - 1) / DW_NC);
  const int nslices = batch_slices(sms, ngroups, (B + DW_BC - 1) / DW_BC);
  return with_const<32, 64, 96, 128>(s.DP, [&](auto DP) {
    constexpr int SB = DP == 128 ? 2 : 4;
    static_assert(dx_smem_bytes(DP, SB) + 1024 <= SMEM_CAP, "dx shared memory");
    if (int r = launch("ctr_residual_unit_bwd(dx, wgmma)", resunit_bwd_dx_wgmma_kernel<DP, SB>, grid, NTHREADS,
                       dx_smem_bytes(DP, SB) + 1024, st, m0, m2, m3, x, b0, out, g_out, d_x, hbuf, ghbuf, d_b1, (int)B,
                       (int)d, (int)H, (int)s.HP))
      return r;
    const int sb = stages_that_fit(1024, dw_smem_bytes(DP, 1));
    const size_t smem = dw_smem_bytes(DP, sb) + 1024;
    if (int r = launch("ctr_residual_unit_bwd(dw1, wgmma)", resunit_bwd_dw_wgmma_kernel<DP, 0>, ngroups * nslices, NTHREADS,
                       smem, st, mh, g_out, out, d_w1, nullptr, (int)B, (int)d, (int)H, ngroups, nslices, sb))
      return r;
    return launch("ctr_residual_unit_bwd(dw0, wgmma)", resunit_bwd_dw_wgmma_kernel<DP, 1>, ngroups * nslices, NTHREADS, smem,
                  st, mgh, x, nullptr, d_w0, d_b0, (int)B, (int)d, (int)H, ngroups, nslices, sb);
  });
}

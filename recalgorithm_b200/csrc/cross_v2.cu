// DCN-V2 cross network (Wang et al., WWW 2021, arXiv:2008.13535, eq. 1-2), row-vector form, l = 0 .. L-1:
//
//   x_{l+1} = x0 o z_l + x_l,   z_l = x_l . W_l + b_l,   x_0 = xl_in (or x0),  out = x_L
//   full rank  W_l = w[l]            w (L,d,d)
//   low rank   W_l = w[l] . u[l]     w (L,d,r), u (L,r,d),  t_l = x_l . w[l]
//
// Backward, g = dL/dx_{l+1} (g_out for l = L-1):  dz = g o x0,  dx0 += g o z_l,
//   full rank  dx_l = g + dz . w[l]^T,              dW_l = x_l^T dz,   db_l = sum_b dz;
//   low rank   dt = dz . u[l]^T, dx_l = g + dt . w[l]^T,   du_l = t_l^T dz (db_l as above),  dw_l = x_l^T dt.
// dx_0 goes to dxl_in, or into dx0 when x_0 = x0.
//
// H100 mapping (3xTF32 wgmma, one TMA producer warp, two consumer warpgroups).  Every GEMM of the layer is one
// K-sliced row GEMM (tc::rows::gemm_ks, as PLE): per 64-sample tile, the tile's A rows (width up to 512, any alignment) are
// staged once in shared memory with ordinary loads, and the operand streams by TMA as a prepped tf32 hi | lo copy, one
// [128 units x 32 inputs] ring stage at a time, each warpgroup taking 64 of the units.  The output goes N-slice by N-slice
// (128 columns) through an epilogue in registers:
//   cross_v2_rows_wgmma_kernel  forward    A = x_l; epilogue z = acc + b, x_{l+1} = x0 o z + x_l (x0, x_l read at the
//                                          accumulator positions); z and x_{l+1} out.  Low rank: a first GEMM
//                                          t = x_l . w[l] (r <= 128: one slice) whose result replaces the staged rows and
//                                          is the A of z = t . u[l] + b, so t only reaches HBM as the saved copy.
//                               backward   A = dz = g o x0, formed while staging and written to the workspace by the
//                                          tile's first CTA; epilogue dx_l = g + acc, dx0 (+)= g o z_l.  Low rank: first
//                                          dt = dz . u[l]^T into the workspace, then A = dt for dx_l.
//   dW, du, dw, db               tc_ptx.cuh's weight_grad_wgmma_kernel (cross_v2::Rows): batch-sliced reductions over the
//                                workspace rows dz / dt with x_l or t_l generated on chip, db as the row sums of dz.
//   cross_v2_prep_kernel         the tf32 hi | lo operand copies of every layer, transposed for the forward.
// One launch per layer and GEMM: a 512-wide tile's x_{l+1} does not fit on chip next to its x_l.  A batch of fewer tiles
// than SMs splits the N-slices of each tile over several CTAs.
//
// Bounds: 1 <= d <= 512, 1 <= L <= 8, 0 <= rank <= 128 (0 = full rank), any B >= 0.
#include <algorithm>

#include "tc_ptx.cuh"

namespace ctr {
namespace cross_v2 {
using namespace ctr::tc;
using namespace ctr::tc::rows;

constexpr int TM = WG_M;                     // samples per tile: both warpgroups share the tile's rows
constexpr int NW = 64;                       // output columns per warpgroup and slice
constexpr int SLICE = NWG * NW;              // output columns per slice: the units of one ring stage
constexpr int SBYTES = ks_stage_bytes<NW>();
constexpr int MAX_D = 512, MAX_L = 8, MAX_R = 128;
constexpr int SU = 16;                       // staging: elements per thread loaded before they are stored

// One launch: A rows (B, lda) [o a_mul], columns < ka, zero padded to the first GEMM's width, times the operand(s).  The
// pointers x_l / out may alias (a forward without `saved` runs in place with nsplit = 1), so none is __restrict__ and the
// rows are read with ordinary loads.
struct Args {                                // the epilogue fields as tc_ptx.cuh's cross_epilogue reads them
  const float* a;
  const float* a_mul;        // A = a o a_mul (dz = g o x0), or null
  float* a_copy;             // the staged A rows (pitch: the first GEMM's KP) written out by each tile's first CTA, or null
  int lda, ka;
  int pre_KP, pre_NP;        // low-rank forward: t = A . pre operand first (pre_KP = 0: none); t is then the main A
  float* t_out;              // t (B, r) written out, or null
  int r;
  int KP, NP, n_slices;      // main GEMM: A width (padded to 32), operand units (padded to SLICE), output slices
  int epi;
  float* y;                  // STORE: y (B, ldy) = acc;  FWD: x_{l+1} (B, d);  BWD: dx_l (B, d), or null
  int ldy;
  const float* bias;         // FWD: b_l
  const float* x0;           // FWD, BWD
  const float* xl;           // FWD: x_l
  float* z_out;              // FWD: z_l, or null
  const float* g;            // BWD: dL/dx_{l+1}
  const float* z;            // BWD: z_l
  float* dx0;                // BWD
  int dx0_accumulate;        // BWD: dx0 += ... (else dx0 = ...)
  int dx0_add_dx;            // BWD: dx_l is added into dx0 instead of being written to y (x_0 = x0)
  int B, d, nsplit, SB;
};

__host__ __device__ constexpr int tile_ld(int KP) { return KP + 4; }   // staged rows: conflict-free A-fragment reads
__host__ __device__ constexpr int smem_bytes(int KP, int SB) { return SB * SBYTES + TM * tile_ld(KP) * 4 + 16 * SB; }

// Writes the tf32 hi | lo copy [2 NP][KP] of the operand of layer blockIdx.y: element (n, k) is src[k][n] (trans) or
// src[n][k] of the layer's rows x cols matrix, 0 outside it.
__global__ void cross_v2_prep_kernel(const float* __restrict__ src, float* __restrict__ dst, int rows, int cols, int trans,
                                     int NP, int KP) {
  const size_t total = (size_t)NP * KP;
  src += (size_t)blockIdx.y * rows * cols;
  dst += (size_t)blockIdx.y * 2 * total;
  const int nu = trans ? cols : rows, nk = trans ? rows : cols;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / KP), k = (int)(idx % KP);
    const float v = (n < nu && k < nk) ? __ldg(src + (trans ? (size_t)k * cols + n : (size_t)n * cols + k)) : 0.f;
    const float hi = tf32_rna(v);
    dst[idx] = hi;                            // hi | lo, with lo rounded to tf32 too (the tensor core would truncate it)
    dst[total + idx] = tf32_rna(v - hi);
  }
}

__global__ void __launch_bounds__(NTHREADS, 1)
cross_v2_rows_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_pre, const __grid_constant__ CUtensorMap tmap,
                           const Args p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  const int KP0 = p.pre_KP ? p.pre_KP : p.KP;                    // width of the staged rows
  const int ld = tile_ld(KP0 > p.KP ? KP0 : p.KP);
  float* xs = reinterpret_cast<float*>(smem + p.SB * SBYTES);   // [64][ld]  A rows (then t)
  const uint32_t sbase = smem_u32(smem);
  Ring ring(smem_u32(xs + TM * ld), p.SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_work = (p.B + TM - 1) / TM * p.nsplit;
  ring.init();
  // ============================ TMA producer: the pre operand, then every slice of the main operand ============================
  if (producer_role(warp, lane, [&] {
        for (int wk = blockIdx.x; wk < n_work; wk += gridDim.x) {
          int s_beg, s_end;
          batch_slice(wk % p.nsplit, p.nsplit, p.n_slices, s_beg, s_end);
          for (int kb = 0; kb < p.pre_KP / KB; ++kb) {
            const Ring::Slot slot = ring.acquire(SBYTES);
            load_ks_stage<NW>(sbase + slot.stage * SBYTES, &tmap_pre, 0, kb, p.pre_NP, slot.full);
          }
          for (int s = s_beg; s < s_end; ++s)
            for (int kb = 0; kb < p.KP / KB; ++kb) {
              const Ring::Slot slot = ring.acquire(SBYTES);
              load_ks_stage<NW>(sbase + slot.stage * SBYTES, &tmap, s * SLICE, kb, p.NP, slot.full);
            }
        }
      }))
    return;

  // ============================ consumers ============================
  const int wg = warp >> 2, w = warp & 3, g = lane >> 2, t = lane & 3;
  const int r0 = w * 16 + g;
  for (int wk = blockIdx.x; wk < n_work; wk += gridDim.x) {
    const int split = wk % p.nsplit;
    int s_beg, s_end;
    batch_slice(split, p.nsplit, p.n_slices, s_beg, s_end);
    const long long base = (long long)(wk / p.nsplit) * TM;
    for (int i0 = threadIdx.x; i0 < TM * KP0; i0 += NWG * 128 * SU) {
      float v[SU];                            // SU loads in flight before the first store
#pragma unroll
      for (int q = 0; q < SU; ++q) {
        const int idx = i0 + q * NWG * 128, r = idx / KP0, c = idx % KP0;
        v[q] = 0.f;
        if (idx < TM * KP0 && c < p.ka && base + r < p.B) {
          const size_t o = (size_t)(base + r) * p.lda + c;
          v[q] = p.a_mul != nullptr ? p.a[o] * p.a_mul[o] : p.a[o];
        }
      }
#pragma unroll
      for (int q = 0; q < SU; ++q) {
        const int idx = i0 + q * NWG * 128, r = idx / KP0, c = idx % KP0;
        if (idx >= TM * KP0) break;
        xs[r * ld + c] = v[q];
        if (p.a_copy != nullptr && split == 0 && base + r < p.B) p.a_copy[(size_t)(base + r) * KP0 + c] = v[q];
      }
    }
    consumers_bar();
    if (p.pre_KP) {                           // t = x_l . w[l] replaces the staged rows once both warpgroups are done
      float acc[NW / 2];
      gemm_ks<NW>(acc, xs, ld, p.pre_KP / KB, r0, t, lane, wg, ring, sbase);
      consumers_bar();
#pragma unroll
      for (int k = 0; k < NW / 2; ++k) {
        const int col = wg * NW + 8 * (k >> 2) + 2 * t + (k & 1), r = r0 + 8 * ((k >> 1) & 1);
        if (col < p.KP) xs[r * ld + col] = acc[k];
        if (p.t_out != nullptr && split == 0 && col < p.r && base + r < p.B) p.t_out[(size_t)(base + r) * p.r + col] = acc[k];
      }
      consumers_bar();
    }
    for (int s = s_beg; s < s_end; ++s) {
      float acc[NW / 2];
      gemm_ks<NW>(acc, xs, ld, p.KP / KB, r0, t, lane, wg, ring, sbase);
      cross_epilogue<NW>(p, acc, base, r0, s * SLICE + wg * NW + 2 * t);
    }
    consumers_bar();                          // the rows may be restaged once every thread has read them
  }
}

// Result rows of tc::weight_grad_wgmma_kernel: row n < n_rows is dst[k * stride + n] over the inputs k, with its batch sum
// in bias[n] when bias is given.  dW_l / du_l: P = dz, rows n = output column, stride d, bias = db_l; dw_l: P = dt, rows
// n = rank column, stride r, no bias.
struct Rows {
  static constexpr bool row_sums = true, mask_q = false, slice_d = true;
  float* dst;
  float* bias;
  int n_rows, stride;
  __device__ __forceinline__ GradRow row(int n) const {
    return n < n_rows ? GradRow{dst + n, stride, bias == nullptr ? nullptr : bias + n} : GradRow{};
  }
};

}  // namespace cross_v2
}  // namespace ctr

// ------------------------------------------------------------------------------------------------ host
using namespace ctr;
using namespace ctr::cross_v2;

namespace {

// Sizes of one call.  Operands per layer (hi | lo, [2 NP][KP]): full rank one of [2 NPd][DP]; low rank one of [2 SLICE][DP]
// (the r units) and one of [2 NPd][RP].  The forward preps the transposed copies, the backward the straight ones, into the
// same workspace bytes.
struct Shape {
  int d, L, r, DP, RP, NPd;
  int64_t op0_floats, op1_floats;            // per layer
  int64_t weight_bytes;                      // every layer's operands: the forward's workspace
  int64_t dz_off, dt_off, g_off[2], bwd_bytes;
  int64_t saved_bytes;
};

int shape_of(const char* fn, int64_t B, int64_t d, int64_t L, int64_t rank, Shape& s) {
  CTR_REQUIRE(B >= 0, "%s: bad batch B=%lld", fn, (long long)B);
  CTR_UNSUPPORTED(d < 1 || d > MAX_D, "%s: unsupported width d=%lld (the tensor-core kernels take 1 <= d <= %d)", fn,
                  (long long)d, MAX_D);
  CTR_UNSUPPORTED(L < 1 || L > MAX_L, "%s: unsupported number of layers L=%lld (1 <= L <= %d)", fn, (long long)L, MAX_L);
  CTR_UNSUPPORTED(rank < 0 || rank > MAX_R, "%s: unsupported rank=%lld (0 <= rank <= %d; 0 = full rank)", fn,
                  (long long)rank, MAX_R);
  CTR_UNSUPPORTED(B > 0x7fffff00LL, "%s: batch too large (B=%lld)", fn, (long long)B);
  s.d = (int)d; s.L = (int)L; s.r = (int)rank;
  s.DP = (int)pad_to(d, KB);
  s.RP = (int)pad_to(rank, KB);
  s.NPd = (int)pad_to(d, SLICE);
  s.op0_floats = rank ? 2LL * SLICE * s.DP : 2LL * s.NPd * s.DP;
  s.op1_floats = rank ? 2LL * s.NPd * s.RP : 0;
  s.weight_bytes = pad_to(L * (s.op0_floats + s.op1_floats) * 4, 128);
  s.dz_off = s.weight_bytes;
  s.dt_off = s.dz_off + pad_to(B * s.DP * 4, 128);
  s.g_off[0] = s.dt_off + pad_to(B * s.RP * 4, 128);
  s.g_off[1] = s.g_off[0] + (L >= 2 ? pad_to(B * d * 4, 128) : 0);
  s.bwd_bytes = s.g_off[1] + (L >= 3 ? pad_to(B * d * 4, 128) : 0);
  s.saved_bytes = B * ((2 * L - 1) * d + L * rank) * 4;
  return CTR_OK;
}

float* at(void* base, int64_t off) { return reinterpret_cast<float*>(static_cast<uint8_t*>(base) + off); }

// one operand of every layer: src (L, rows, cols) -> [2 NP][KP] per layer at dst
int prep(const char* what, const float* src, float* dst, int rows, int cols, int trans, int NP, int KP, int L,
         cudaStream_t st) {
  return launch(what, cross_v2_prep_kernel, dim3(capped_grid(((int64_t)NP * KP + 255) / 256, 256), L), 256, 0, st, src, dst,
                rows, cols, trans, NP, KP);
}

// The rows kernel over B samples with the operand map of layer-operand `op` ([2 NP][KP] at op) and, for the low-rank
// forward, the pre operand `pre`.  `in_place`: the output overwrites the staged input, so each tile stays in one CTA.
int rows_gemm(const char* fn, const char* what, Args a, const float* pre, const float* op, bool in_place, cudaStream_t st) {
  CUtensorMap mpre, mop;
  int rc;
  if ((rc = encode_2d(fn, &mop, op, a.KP, 2 * (int64_t)a.NP, KB, SLICE, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  mpre = mop;
  if (pre != nullptr && (rc = encode_2d(fn, &mpre, pre, a.pre_KP, 2 * (int64_t)a.pre_NP, KB, SLICE, CU_TENSOR_MAP_SWIZZLE_128B)))
    return rc;
  const int sms = sm_count();
  const int64_t n_tiles = (a.B + TM - 1) / TM;
  a.nsplit = in_place ? 1 : (int)std::max<int64_t>(1, std::min<int64_t>(sms / n_tiles, a.n_slices));
  const int KPmax = std::max(a.pre_KP ? a.pre_KP : a.KP, a.KP);
  a.SB = std::min<int>(4, (int)((SMEM_CAP - 1024 - smem_bytes(KPmax, 0)) / (SBYTES + 16)));
  return launch(what, cross_v2_rows_wgmma_kernel, capped_grid(n_tiles * a.nsplit, sms), NTHREADS,
                smem_bytes(KPmax, a.SB) + 1024, st, mpre, mop, a);
}
static_assert(smem_bytes(MAX_D, 2) + 1024 <= (int)SMEM_CAP, "rows kernel shared memory at the bounds");

// N of the weight-gradient kernel for inputs of width q: the 32 / 64 / 128 class, 128 with slices past 128
int dw_n(int q) { return q <= 128 ? pad3(q) : 128; }

int weight_grad(const char* fn, const char* what, const Rows& rows, const float* p, int64_t units, int64_t B, const float* q,
                int qd, cudaStream_t st) {
  const int N = dw_n(qd);
  return with_const<32, 64, 128>(N, [&](auto n) {
    return launch_weight_grad<n>(fn, what, rows, p, units, B, q, nullptr, qd, (qd + N - 1) / N, st);
  });
}

}  // namespace

extern "C" int ctr_cross_v2_workspace_bytes(int64_t B, int64_t d, int64_t L, int64_t rank, int64_t* workspace_bytes,
                                            int64_t* saved_bytes) {
  static const char* fn = "ctr_cross_v2_workspace_bytes";
  CTR_REQUIRE(workspace_bytes != nullptr && saved_bytes != nullptr, "%s: null argument", fn);
  Shape s;
  if (int rc = shape_of(fn, B, d, L, rank, s)) return rc;
  *workspace_bytes = s.bwd_bytes;
  *saved_bytes = s.saved_bytes;
  return CTR_OK;
}

extern "C" int ctr_cross_v2_fwd(const float* x0, const float* xl_in, const float* w, const float* u, const float* b,
                                int64_t B, int64_t d, int64_t L, int64_t rank, float* out, void* saved, void* workspace,
                                int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_cross_v2_fwd";
  Shape s;
  int rc = shape_of(fn, B, d, L, rank, s);
  if (rc) return rc;
  CTR_REQUIRE(x0 && w && b && out && (rank == 0 || u), "ctr_cross_v2_fwd: null argument");
  if ((rc = check_workspace(fn, "ctr_cross_v2_workspace_bytes with B = 0", workspace, workspace_bytes, s.weight_bytes)))
    return rc;
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  float* op0 = static_cast<float*>(workspace);
  float* op1 = op0 + L * s.op0_floats;
  if (rank == 0) {
    rc = prep("ctr_cross_v2_fwd(prep)", w, op0, s.d, s.d, 1, s.NPd, s.DP, s.L, st);
  } else if (!(rc = prep("ctr_cross_v2_fwd(prep w)", w, op0, s.d, s.r, 1, SLICE, s.DP, s.L, st))) {
    rc = prep("ctr_cross_v2_fwd(prep u)", u, op1, s.r, s.d, 1, s.NPd, s.RP, s.L, st);
  }
  if (rc) return rc;
  // saved: x_1 .. x_{L-1}, then z_0 .. z_{L-1}, then t_0 .. t_{L-1} (low rank)
  float* xs = static_cast<float*>(saved);
  float* zs = xs == nullptr ? nullptr : xs + (L - 1) * B * d;
  float* ts = xs == nullptr ? nullptr : zs + L * B * d;
  for (int l = 0; l < s.L; ++l) {
    const float* xl = l == 0 ? (xl_in ? xl_in : x0) : (xs ? xs + (l - 1) * B * d : out);
    Args a = {};
    a.a = xl; a.lda = s.d; a.ka = s.d;
    a.epi = EPI_FWD; a.y = l == s.L - 1 || xs == nullptr ? out : xs + l * B * d;
    a.bias = b + (size_t)l * d; a.x0 = x0; a.xl = xl; a.z_out = zs ? zs + l * B * d : nullptr;
    a.NP = s.NPd; a.n_slices = s.NPd / SLICE; a.B = (int)B; a.d = s.d;
    const float* pre = nullptr;
    const float* op = op0 + l * s.op0_floats;
    if (rank == 0) {
      a.KP = s.DP;
    } else {
      a.pre_KP = s.DP; a.pre_NP = SLICE; a.t_out = ts ? ts + l * B * rank : nullptr; a.r = s.r;
      a.KP = s.RP;
      pre = op;
      op = op1 + l * s.op1_floats;
    }
    if ((rc = rows_gemm(fn, "ctr_cross_v2_fwd(wgmma)", a, pre, op, xl == out, st))) return rc;
  }
  return CTR_OK;
}

extern "C" int ctr_cross_v2_bwd(const float* x0, const float* xl_in, const float* w, const float* u, const float* b,
                                const void* saved, const float* g_out, int64_t B, int64_t d, int64_t L, int64_t rank,
                                float* dx0, float* dxl_in, float* dw, float* du, float* db, void* workspace,
                                int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_cross_v2_bwd";
  Shape s;
  int rc = shape_of(fn, B, d, L, rank, s);
  if (rc) return rc;
  CTR_REQUIRE(x0 && w && b && saved && g_out && dx0 && dw && db && (rank == 0 || (u && du)) && (!xl_in || dxl_in),
              "ctr_cross_v2_bwd: null argument");
  if ((rc = check_workspace(fn, "ctr_cross_v2_workspace_bytes", workspace, workspace_bytes, s.bwd_bytes))) return rc;
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)(L * d * (rank ? rank : d)), st));
  if (rank) CTR_CUDA(cudaMemsetAsync(du, 0, sizeof(float) * (size_t)(L * rank * d), st));
  CTR_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * (size_t)(L * d), st));
  if (B == 0) return CTR_OK;
  float* op0 = static_cast<float*>(workspace);
  float* op1 = op0 + L * s.op0_floats;
  if (rank == 0) {
    rc = prep("ctr_cross_v2_bwd(prep)", w, op0, s.d, s.d, 0, s.NPd, s.DP, s.L, st);
  } else if (!(rc = prep("ctr_cross_v2_bwd(prep u)", u, op0, s.r, s.d, 0, SLICE, s.DP, s.L, st))) {
    rc = prep("ctr_cross_v2_bwd(prep w)", w, op1, s.d, s.r, 0, s.NPd, s.RP, s.L, st);
  }
  if (rc) return rc;
  const float* xs = static_cast<const float*>(saved);
  const float* zs = xs + (L - 1) * B * d;
  const float* ts = zs + L * B * d;
  float* dz = at(workspace, s.dz_off);
  float* dt = at(workspace, s.dt_off);
  const float* g = g_out;
  for (int l = s.L - 1; l >= 0; --l) {
    const float* xl = l == 0 ? (xl_in ? xl_in : x0) : xs + (l - 1) * B * d;
    float* gnext = l == 0 ? (xl_in ? dxl_in : nullptr) : at(workspace, s.g_off[(s.L - 1 - l) & 1]);
    Args a = {};
    a.a = g; a.a_mul = x0; a.a_copy = dz; a.lda = s.d; a.ka = s.d; a.KP = s.DP;
    a.B = (int)B; a.d = s.d;
    if (rank) {                               // dt = dz . u[l]^T, then A = dt
      a.NP = SLICE; a.n_slices = 1; a.epi = EPI_STORE; a.y = dt; a.ldy = s.RP;
      if ((rc = rows_gemm(fn, "ctr_cross_v2_bwd(dt, wgmma)", a, nullptr, op0 + l * s.op0_floats, false, st))) return rc;
      a.a = dt; a.a_mul = nullptr; a.a_copy = nullptr; a.lda = s.RP; a.ka = s.RP; a.KP = s.RP;
    }
    a.NP = s.NPd; a.n_slices = s.NPd / SLICE; a.epi = EPI_BWD; a.y = gnext; a.ldy = 0;
    a.g = g; a.z = zs + l * B * d; a.x0 = x0; a.dx0 = dx0; a.dx0_accumulate = l < s.L - 1; a.dx0_add_dx = l == 0 && !xl_in;
    if ((rc = rows_gemm(fn, "ctr_cross_v2_bwd(dx, wgmma)", a, nullptr, rank ? op1 + l * s.op1_floats : op0 + l * s.op0_floats,
                        false, st)))
      return rc;
    float* dbl = db + (size_t)l * d;
    if (rank == 0) {
      rc = weight_grad(fn, "ctr_cross_v2_bwd(dw, wgmma)", Rows{dw + (size_t)l * d * d, dbl, s.d, s.d}, dz, s.DP, B, xl, s.d, st);
    } else if (!(rc = weight_grad(fn, "ctr_cross_v2_bwd(du, wgmma)", Rows{du + (size_t)l * rank * d, dbl, s.d, s.d}, dz, s.DP,
                                  B, ts + l * B * rank, s.r, st))) {
      rc = weight_grad(fn, "ctr_cross_v2_bwd(dw, wgmma)", Rows{dw + (size_t)l * d * rank, nullptr, s.r, s.r}, dt, s.RP, B, xl,
                       s.d, st);
    }
    if (rc) return rc;
    g = gnext;
  }
  return CTR_OK;
}

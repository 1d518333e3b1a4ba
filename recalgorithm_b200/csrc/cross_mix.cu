// DCN-Mix cross network: a mixture of low-rank cross experts (Wang et al., WWW 2021, arXiv:2008.13535, eq. 3-4), row-vector
// form, l = 0 .. L-1, experts i = 1 .. K, x_0 = x0, out = x_L, g = tanh or the identity:
//
//   q_i = x_l . v[l,i],  t_i = g(q_i),  m_i = t_i . c[l,i],  c~_i = g(m_i)      v (L,K,d,r), c (L,K,r,r)
//   p = softmax_i(x_l . gate)                                                   gate (d,K), shared by the layers
//   z_l = sum_i p_i c~_i . u[l,i] + b[l],   x_{l+1} = x0 o z_l + x_l             u (L,K,r,d), b (L,d)
//
// The paper's sum_i p_i (x0 o (c~_i u_i + b)) equals x0 o z_l since sum_i p_i = 1; the kernels compute this collapsed form:
// with the experts side by side (K r <= 128 columns), q = x_l . [v_1 .. v_K], m = t . blockdiag(c) and
// z_l = [p_1 c~_1 | .. | p_K c~_K] . [u_1; ..; u_K] + b.
//
// Backward, G = dL/dx_{l+1}:  dz = G o x0,  dx0 += G o z_l,  db_l = sum_b dz,  e = dz . [u]^T,  dp_i = <c~_i, e_i>,
//   ds_i = p_i (dp_i - sum_j p_j dp_j),  dm_i = p_i e_i o g'(m_i),  dq_i = (dm_i . c[l,i]^T) o g'(q_i),
//   dx_l = G + [dq | ds] . [v | gate]^T;   du = (p c~)^T dz,  dc_i = t_i^T dm_i,  dv = x_l^T dq,  dgate += x_l^T ds.
// dx_0 is added into dx0.
//
// H100 mapping: DCN-V2's (cross_v2.cu) K-sliced 3xTF32 row GEMMs (tc::rows::gemm_ks) over 64-sample tiles, with one TMA
// producer warp and two consumer warpgroups; each operand is a prepped tf32 hi | lo copy.  One kernel, three modes:
//   FWD        stage x_l; the K gate logits per row on the CUDA cores from the staged rows, softmax -> p (shared memory);
//              t = g(x_l . [v]) (one 128-unit slice) replaces the staged rows; c~ = g(t . blockdiag(c)) (one slice, the
//              prep writes the zero off-diagonal blocks); a = p o c~ replaces the staged rows; then a . [u] over the
//              N-slices of d with DCN-V2's forward epilogue.  t, c~ and p go to `saved`.
//   BWD_CHAIN  stage dz = G o x0 (written to the workspace); e = dz . [u]^T (one slice) into shared memory; dp, ds, dm and
//              a = p o c~ from it on the CUDA cores (per-row sums over K r columns span both warpgroups, so they run out of
//              shared memory, not registers); dm replaces the staged rows; dq = (dm . blockdiag(c)^T) o g'(q).  Writes a,
//              dm and [dq | ds] to the workspace.
//   BWD_DX     stage [dq | ds]; times [v | gate]^T over the N-slices of d with DCN-V2's backward epilogue.
// The weight gradients run on tc_ptx.cuh's weight_grad_wgmma_kernel (cross_mix::Rows): du with db as its row sums
// (P = dz, Q = a); dv and dgate in one launch (P = [dq | ds], Q = x_l; the rows past K r go to dgate, accumulated over the
// layers); dc as the full (K r)^2 t^T dm reduction into the workspace, whose diagonal blocks cross_mix_fold_kernel copies.
//
// Bounds: 1 <= d <= 512, 1 <= L <= 8, 1 <= K <= 16, r >= 1, K r <= 128, any B >= 0.
#include <algorithm>

#include "tc_ptx.cuh"

namespace ctr {
namespace cross_mix {
using namespace ctr::tc;
using namespace ctr::tc::rows;

constexpr int TM = WG_M;                     // samples per tile: both warpgroups share the tile's rows
constexpr int NW = 64;                       // output columns per warpgroup and slice
constexpr int SLICE = NWG * NW;              // output columns per slice: the units of one ring stage
constexpr int SBYTES = ks_stage_bytes<NW>();
constexpr int MAX_D = 512, MAX_L = 8, MAX_K = 16, MAX_KR = SLICE;
constexpr int SU = 16;                       // staging: elements per thread loaded before they are stored

enum Mode { FWD = 0, BWD_CHAIN = 1, BWD_DX = 2 };

// One launch.  The pointers x_l / out may alias (a forward without `saved` runs in place with nsplit = 1), so none is
// __restrict__ and the rows are read with ordinary loads.
struct Args {                                // the epilogue fields as tc_ptx.cuh's cross_epilogue reads them
  int mode, act;                             // act: 1 tanh, 0 identity
  const float* a;                            // staged rows: A = a o a_mul (B, lda), columns < ka, zero padded to KP0
  const float* a_mul;
  float* a_copy;                             // the staged rows (pitch KP0) written out by each tile's first CTA, or null
  int lda, ka, KP0;
  int K, r, KR, KRP;                         // experts, rank, K r and K r padded to 32 (FWD, BWD_CHAIN)
  const float* gate;                         // FWD: (d, K)
  float* t;                                  // saved t (B, KR): FWD writes it (or null), BWD_CHAIN reads it
  float* ct;                                 // saved c~ (B, KR), as t
  float* pg;                                 // saved p (B, K), as t
  float* a_out;                              // BWD_CHAIN: p o c~ (B, KR)
  float* dm_out;                             // BWD_CHAIN: dm (B, KRP)
  float* w_out;                              // BWD_CHAIN: [dq | ds] (B, ldw)
  int ldw;
  int KP, NP, n_slices;                      // main GEMM (FWD, BWD_DX): A width, operand units, output slices
  int epi;
  float* y;                                  // FWD: x_{l+1} (B, d);  BWD: dx_l (B, d), or null
  int ldy;
  const float* bias;                         // FWD: b_l
  const float* x0;                           // FWD, BWD
  const float* xl;                           // FWD: x_l
  float* z_out;                              // FWD: z_l, or null
  const float* g;                            // BWD: dL/dx_{l+1}
  const float* z;                            // BWD: z_l
  float* dx0;                                // BWD
  int dx0_accumulate;                        // BWD: dx0 += ... (else dx0 = ...)
  int dx0_add_dx;                            // BWD: dx_l is added into dx0 instead of being written to y (l = 0)
  int B, d, nsplit, SB;
};

__host__ __device__ constexpr int tile_ld(int KP) { return KP + 4; }   // staged rows: conflict-free A-fragment reads
// ring stages, the staged rows (width KPmax), the per-row gate values sg / sp [64][MAX_K] and the ring barriers
__host__ __device__ constexpr int smem_bytes(int KPmax, int SB) {
  return SB * SBYTES + TM * tile_ld(KPmax) * 4 + 2 * TM * MAX_K * 4 + 16 * SB;
}

__device__ __forceinline__ float act_fn(float v, int act) { return act ? tanhf(v) : v; }

// The operands, as [2 NP][KP] tf32 hi | lo copies per layer: element (n, k) multiplies A column k into output column n.
enum Op {
  OP_V = 0,    // FWD   q:   (i r + j, k)       = v[l,i,k,j]
  OP_C = 1,    // FWD   m:   (i r + j', i r + j) = c[l,i,j,j'], 0 off the diagonal blocks
  OP_U = 2,    // FWD   z:   (n, i r + j)       = u[l,i,j,n]
  OP_UT = 3,   // BWD   e:   (i r + j, n)       = u[l,i,j,n]
  OP_CT = 4,   // BWD   dq:  (i r + j, i r + j') = c[l,i,j,j'], 0 off the diagonal blocks
  OP_VG = 5    // BWD   dx:  (n, i r + j)       = v[l,i,n,j];  (n, K r + i) = gate[n,i]
};

// Writes the tf32 hi | lo copy [2 NP][KP] of operand `op` of layer blockIdx.y, layer_floats apart (0 outside the operand).
__global__ void cross_mix_prep_kernel(const float* __restrict__ src, const float* __restrict__ gate, float* __restrict__ dst,
                                      int64_t layer_floats, int op, int d, int K, int r, int NP, int KP) {
  const size_t total = (size_t)NP * KP;
  const int l = blockIdx.y, KR = K * r;
  dst += (size_t)l * layer_floats;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / KP), k = (int)(idx % KP);
    float v = 0.f;
    switch (op) {
      case OP_V:
        if (n < KR && k < d) v = __ldg(src + (((size_t)l * K + n / r) * d + k) * r + n % r);
        break;
      case OP_C:
        if (n < KR && k < KR && n / r == k / r) v = __ldg(src + (((size_t)l * K + n / r) * r + k % r) * r + n % r);
        break;
      case OP_U:
        if (n < d && k < KR) v = __ldg(src + (((size_t)l * K + k / r) * r + k % r) * d + n);
        break;
      case OP_UT:
        if (n < KR && k < d) v = __ldg(src + (((size_t)l * K + n / r) * r + n % r) * d + k);
        break;
      case OP_CT:
        if (n < KR && k < KR && n / r == k / r) v = __ldg(src + (((size_t)l * K + n / r) * r + n % r) * r + k % r);
        break;
      default:  // OP_VG
        if (n < d && k < KR) v = __ldg(src + (((size_t)l * K + k / r) * d + n) * r + k % r);
        else if (n < d && k < KR + K) v = __ldg(gate + (size_t)n * K + (k - KR));
    }
    const float hi = tf32_rna(v);
    dst[idx] = hi;                            // hi | lo, with lo rounded to tf32 too (the tensor core would truncate it)
    dst[total + idx] = tf32_rna(v - hi);
  }
}

__global__ void __launch_bounds__(NTHREADS, 1)
cross_mix_rows_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_pre, const __grid_constant__ CUtensorMap tmap_mid,
                            const __grid_constant__ CUtensorMap tmap, const Args p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align_1024(smem_raw);
  const bool experts = p.mode != BWD_DX;                        // the two expert GEMMs run
  const int ld = tile_ld(p.KP0 > p.KRP ? p.KP0 : p.KRP);
  float* xs = reinterpret_cast<float*>(smem + p.SB * SBYTES);   // [64][ld]  staged rows, then t / e, then a / dm
  float* sg = xs + TM * ld;                                     // [64][MAX_K]  gate logits (FWD), dp (BWD_CHAIN)
  float* sp = sg + TM * MAX_K;                                  // [64][MAX_K]  p
  const uint32_t sbase = smem_u32(smem);
  Ring ring(smem_u32(sp + TM * MAX_K), p.SB);

  const int warp = warp_uniform(threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int n_work = (p.B + TM - 1) / TM * p.nsplit;
  ring.init();
  // ============================ TMA producer: the two expert operands, then every slice of the main operand ============================
  if (producer_role(warp, lane, [&] {
        for (int wk = blockIdx.x; wk < n_work; wk += gridDim.x) {
          int s_beg, s_end;
          batch_slice(wk % p.nsplit, p.nsplit, p.n_slices, s_beg, s_end);
          if (experts) {
            for (int kb = 0; kb < p.KP0 / KB; ++kb) {
              const Ring::Slot slot = ring.acquire(SBYTES);
              load_ks_stage<NW>(sbase + slot.stage * SBYTES, &tmap_pre, 0, kb, SLICE, slot.full);
            }
            for (int kb = 0; kb < p.KRP / KB; ++kb) {
              const Ring::Slot slot = ring.acquire(SBYTES);
              load_ks_stage<NW>(sbase + slot.stage * SBYTES, &tmap_mid, 0, kb, SLICE, slot.full);
            }
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
  const int r0 = w * 16 + g, tid = threadIdx.x;
  for (int wk = blockIdx.x; wk < n_work; wk += gridDim.x) {
    const int split = wk % p.nsplit;
    const bool first = split == 0;            // the tile's CTA that writes its per-sample rows out
    int s_beg, s_end;
    batch_slice(split, p.nsplit, p.n_slices, s_beg, s_end);
    const long long base = (long long)(wk / p.nsplit) * TM;
    for (int i0 = tid; i0 < TM * p.KP0; i0 += NWG * 128 * SU) {
      float v[SU];                            // SU loads in flight before the first store
#pragma unroll
      for (int q = 0; q < SU; ++q) {
        const int idx = i0 + q * NWG * 128, r = idx / p.KP0, c = idx % p.KP0;
        v[q] = 0.f;
        if (idx < TM * p.KP0 && c < p.ka && base + r < p.B) {
          const size_t o = (size_t)(base + r) * p.lda + c;
          v[q] = p.a_mul != nullptr ? p.a[o] * p.a_mul[o] : p.a[o];
        }
      }
#pragma unroll
      for (int q = 0; q < SU; ++q) {
        const int idx = i0 + q * NWG * 128, r = idx / p.KP0, c = idx % p.KP0;
        if (idx >= TM * p.KP0) break;
        xs[r * ld + c] = v[q];
        if (p.a_copy != nullptr && first && base + r < p.B) p.a_copy[(size_t)(base + r) * p.KP0 + c] = v[q];
      }
    }
    consumers_bar();
    if (experts) {
      if (p.mode == FWD) {                    // gate logits, then p = softmax (max subtracted) per row
        for (int idx = tid; idx < TM * p.K; idx += NWG * 128) {
          const int r = idx / p.K, i = idx % p.K;
          const float* xr = xs + r * ld;
          float s[4] = {0.f, 0.f, 0.f, 0.f};  // four chains: the sum is latency bound
          int k = 0;
          for (; k + 4 <= p.d; k += 4) {
#pragma unroll
            for (int q = 0; q < 4; ++q) s[q] = fmaf(xr[k + q], __ldg(p.gate + (size_t)(k + q) * p.K + i), s[q]);
          }
          for (; k < p.d; ++k) s[0] = fmaf(xr[k], __ldg(p.gate + (size_t)k * p.K + i), s[0]);
          sg[r * MAX_K + i] = (s[0] + s[1]) + (s[2] + s[3]);
        }
        consumers_bar();
        if (tid < TM) {
          const int r = tid;
          float mx = sg[r * MAX_K];
          for (int i = 1; i < p.K; ++i) mx = fmaxf(mx, sg[r * MAX_K + i]);
          float sum = 0.f;
          for (int i = 0; i < p.K; ++i) {
            const float e = expf(sg[r * MAX_K + i] - mx);
            sp[r * MAX_K + i] = e;
            sum += e;
          }
          for (int i = 0; i < p.K; ++i) {
            const float pv = sp[r * MAX_K + i] / sum;
            sp[r * MAX_K + i] = pv;
            if (p.pg != nullptr && first && base + r < p.B) p.pg[(size_t)(base + r) * p.K + i] = pv;
          }
        }
      }
      float acc[NW / 2];
      gemm_ks<NW>(acc, xs, ld, p.KP0 / KB, r0, t, lane, wg, ring, sbase);   // FWD: q = x_l . [v];  BWD: e = dz . [u]^T
      consumers_bar();
#pragma unroll
      for (int k = 0; k < NW / 2; ++k) {
        const int col = wg * NW + 8 * (k >> 2) + 2 * t + (k & 1), r = r0 + 8 * ((k >> 1) & 1);
        float v = acc[k];
        if (p.mode == FWD) {
          v = act_fn(v, p.act);
          if (p.t != nullptr && first && col < p.KR && base + r < p.B) p.t[(size_t)(base + r) * p.KR + col] = v;
        }
        if (col < p.KRP) xs[r * ld + col] = v;
      }
      consumers_bar();
      if (p.mode == BWD_CHAIN) {
        for (int idx = tid; idx < TM * p.K; idx += NWG * 128) {      // dp_i = <c~_i, e_i>, and p_i
          const int r = idx / p.K, i = idx % p.K;
          const long long row = base + r;
          float dp = 0.f, pv = 0.f;
          if (row < p.B) {
            const float* cr = p.ct + (size_t)row * p.KR + i * p.r;
            const float* er = xs + r * ld + i * p.r;
            for (int j = 0; j < p.r; ++j) dp = fmaf(cr[j], er[j], dp);
            pv = p.pg[(size_t)row * p.K + i];
          }
          sg[r * MAX_K + i] = dp;
          sp[r * MAX_K + i] = pv;
        }
        consumers_bar();
        if (tid < TM && base + tid < p.B) {   // ds_i = p_i (dp_i - sum_j p_j dp_j)
          const int r = tid;
          float sdp = 0.f;
          for (int i = 0; i < p.K; ++i) sdp = fmaf(sp[r * MAX_K + i], sg[r * MAX_K + i], sdp);
          for (int i = 0; i < p.K; ++i)
            p.w_out[(size_t)(base + r) * p.ldw + p.KR + i] = sp[r * MAX_K + i] * (sg[r * MAX_K + i] - sdp);
        }
        for (int idx = tid; idx < TM * p.KRP; idx += NWG * 128) {    // dm = p e o g'(m), a = p c~
          const int r = idx / p.KRP, c = idx % p.KRP;
          const long long row = base + r;
          float dm = 0.f;
          if (c < p.KR && row < p.B) {
            const float pv = sp[r * MAX_K + c / p.r], cv = p.ct[(size_t)row * p.KR + c];
            dm = pv * xs[r * ld + c];
            if (p.act) dm *= 1.f - cv * cv;
            p.a_out[(size_t)row * p.KR + c] = pv * cv;
          }
          xs[r * ld + c] = dm;
          if (row < p.B) p.dm_out[(size_t)row * p.KRP + c] = dm;
        }
        consumers_bar();
      }
      gemm_ks<NW>(acc, xs, ld, p.KRP / KB, r0, t, lane, wg, ring, sbase);  // FWD: m = t . bd(c);  BWD: dm . bd(c)^T
      if (p.mode == FWD) {
        consumers_bar();
#pragma unroll
        for (int k = 0; k < NW / 2; ++k) {    // a = p o c~ replaces the staged rows
          const int col = wg * NW + 8 * (k >> 2) + 2 * t + (k & 1), r = r0 + 8 * ((k >> 1) & 1);
          if (col < p.KR) {
            const float cv = act_fn(acc[k], p.act);
            if (p.ct != nullptr && first && base + r < p.B) p.ct[(size_t)(base + r) * p.KR + col] = cv;
            xs[r * ld + col] = sp[r * MAX_K + col / p.r] * cv;
          } else if (col < p.KRP) {
            xs[r * ld + col] = 0.f;
          }
        }
        consumers_bar();
      } else {
#pragma unroll
        for (int k = 0; k < NW / 2; ++k) {    // dq = acc o g'(q)
          const int col = wg * NW + 8 * (k >> 2) + 2 * t + (k & 1), r = r0 + 8 * ((k >> 1) & 1);
          if (col < p.KR && base + r < p.B) {
            const size_t o = (size_t)(base + r);
            float dq = acc[k];
            if (p.act) {
              const float tv = p.t[o * p.KR + col];
              dq *= 1.f - tv * tv;
            }
            p.w_out[o * p.ldw + col] = dq;
          }
        }
      }
    }
    for (int s = s_beg; s < s_end; ++s) {
      float acc[NW / 2];
      gemm_ks<NW>(acc, xs, ld, p.KP / KB, r0, t, lane, wg, ring, sbase);
      cross_epilogue<NW>(p, acc, base, r0, s * SLICE + wg * NW + 2 * t);
    }
    consumers_bar();                          // the rows may be restaged once every thread has read them
  }
}

// dc[l,i,j,j'] = S_l[(i r + j) K r + i r + j']: the diagonal blocks of the full t^T dm reduction S_l (K r, K r)
__global__ void cross_mix_fold_kernel(const float* __restrict__ S, float* __restrict__ dc, int L, int K, int r) {
  const int KR = K * r;
  const int64_t total = (int64_t)L * K * r * r;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int jp = (int)(idx % r), j = (int)(idx / r % r), i = (int)(idx / ((int64_t)r * r) % K);
    const int64_t l = idx / ((int64_t)K * r * r);
    dc[idx] = S[(l * KR + i * r + j) * KR + i * r + jp];
  }
}

// Result rows of tc::weight_grad_wgmma_kernel: row n < n_rows is dst[(n / group) group_pitch + n % group + k stride] over
// the inputs k, with its batch sum in bias[n] when bias is given; row n_rows + i (i < n_tail) is tail[i + k tail_stride].
//   du_l:          P = dz, Q = a = p o c~:  rows n = output column, group = d, stride d, bias db_l;
//   dv_l, dgate:   P = [dq | ds], Q = x_l:  rows i r + j -> dv[l,i,k,j] (group r, pitch d r, stride r), rows K r + i ->
//                  dgate[k,i] (stride K);
//   S_l:           P = dm, Q = t:           rows n = K r column, stride K r.
struct Rows {
  static constexpr bool row_sums = true, mask_q = false, slice_d = true;
  float* dst;
  float* bias;
  int n_rows, group, group_pitch, stride;
  float* tail;
  int n_tail, tail_stride;
  __device__ __forceinline__ GradRow row(int n) const {
    if (n < n_rows)
      return GradRow{dst + (size_t)(n / group) * group_pitch + n % group, stride, bias == nullptr ? nullptr : bias + n};
    return n - n_rows < n_tail ? GradRow{tail + (n - n_rows), tail_stride, nullptr} : GradRow{};
  }
};

}  // namespace cross_mix
}  // namespace ctr

// ------------------------------------------------------------------------------------------------ host
using namespace ctr;
using namespace ctr::cross_mix;

namespace {

// Sizes of one call.  Operands per layer (hi | lo, [2 NP][KP]): pre [2 SLICE][DP] (v, or u^T), mid [2 SLICE][KRP]
// (blockdiag(c), or its transpose), main [2 NPd][W2] (u with KP = KRP, or [v | gate]^T).  The forward preps its copies,
// the backward its own, into the same workspace bytes.
struct Shape {
  int d, L, K, r, KR, DP, KRP, W2, NPd;
  int64_t pre_floats, mid_floats, main_floats;   // per layer
  int64_t weight_bytes;                          // every layer's operands: the forward's workspace
  int64_t dz_off, a_off, dm_off, w_off, s_off, g_off[2], bwd_bytes;
  int64_t saved_bytes;
};

int shape_of(const char* fn, int64_t B, int64_t d, int64_t L, int64_t K, int64_t r, Shape& s) {
  CTR_REQUIRE(B >= 0, "%s: bad batch B=%lld", fn, (long long)B);
  CTR_UNSUPPORTED(d < 1 || d > MAX_D, "%s: unsupported width d=%lld (the tensor-core kernels take 1 <= d <= %d)", fn,
                  (long long)d, MAX_D);
  CTR_UNSUPPORTED(L < 1 || L > MAX_L, "%s: unsupported number of layers L=%lld (1 <= L <= %d)", fn, (long long)L, MAX_L);
  CTR_UNSUPPORTED(K < 1 || K > MAX_K, "%s: unsupported number of experts K=%lld (1 <= K <= %d)", fn, (long long)K, MAX_K);
  CTR_UNSUPPORTED(r < 1 || r > MAX_KR, "%s: unsupported rank r=%lld (r >= 1 and K*r <= %d)", fn, (long long)r, MAX_KR);
  CTR_UNSUPPORTED(K * r > MAX_KR, "%s: unsupported K=%lld experts of rank r=%lld (K*r <= %d)", fn, (long long)K,
                  (long long)r, MAX_KR);
  CTR_UNSUPPORTED(B > 0x7fffff00LL, "%s: batch too large (B=%lld)", fn, (long long)B);
  s.d = (int)d; s.L = (int)L; s.K = (int)K; s.r = (int)r; s.KR = (int)(K * r);
  s.DP = (int)pad_to(d, KB);
  s.KRP = (int)pad_to(s.KR, KB);
  s.W2 = (int)pad_to(s.KR + K, KB);
  s.NPd = (int)pad_to(d, SLICE);
  s.pre_floats = 2LL * SLICE * s.DP;
  s.mid_floats = 2LL * SLICE * s.KRP;
  s.main_floats = 2LL * s.NPd * s.W2;
  s.weight_bytes = pad_to(L * (s.pre_floats + s.mid_floats + s.main_floats) * 4, 128);
  s.dz_off = s.weight_bytes;
  s.a_off = s.dz_off + pad_to(B * s.DP * 4, 128);
  s.dm_off = s.a_off + pad_to(B * s.KR * 4, 128);
  s.w_off = s.dm_off + pad_to(B * s.KRP * 4, 128);
  s.s_off = s.w_off + pad_to(B * s.W2 * 4, 128);
  s.g_off[0] = s.s_off + (B > 0 ? pad_to(L * s.KR * s.KR * 4, 128) : 0);   // the batch-0 backward reduces nothing
  s.g_off[1] = s.g_off[0] + (L >= 2 ? pad_to(B * d * 4, 128) : 0);
  s.bwd_bytes = s.g_off[1] + (L >= 3 ? pad_to(B * d * 4, 128) : 0);
  s.saved_bytes = B * ((2 * L - 1) * d + L * (2 * s.KR + K)) * 4;
  return CTR_OK;
}

float* at(void* base, int64_t off) { return reinterpret_cast<float*>(static_cast<uint8_t*>(base) + off); }

// operand `op` of every layer -> [2 NP][KP] per layer, layer_floats apart, at dst
int prep(const char* what, int op, const float* src, const float* gate, float* dst, int64_t layer_floats, int NP, int KP,
         const Shape& s, cudaStream_t st) {
  return launch(what, cross_mix_prep_kernel, dim3(capped_grid(((int64_t)NP * KP + 255) / 256, 256), s.L), 256, 0, st, src,
                gate, dst, layer_floats, op, s.d, s.K, s.r, NP, KP);
}

// The rows kernel over B samples.  pre / mid: the expert operands ([2 SLICE][KP0], [2 SLICE][KRP]; FWD and BWD_CHAIN);
// op: the main operand ([2 NP][KP]; FWD and BWD_DX).  `in_place`: the output overwrites the staged input, so each tile
// stays in one CTA.
int rows_gemm(const char* fn, const char* what, Args a, const float* pre, const float* mid, const float* op, bool in_place,
              cudaStream_t st) {
  CUtensorMap mpre{}, mmid{}, mop{};
  int rc;
  if (op != nullptr && (rc = encode_2d(fn, &mop, op, a.KP, 2 * (int64_t)a.NP, KB, SLICE, CU_TENSOR_MAP_SWIZZLE_128B)))
    return rc;
  if (pre != nullptr) {
    if ((rc = encode_2d(fn, &mpre, pre, a.KP0, 2 * (int64_t)SLICE, KB, SLICE, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
    if ((rc = encode_2d(fn, &mmid, mid, a.KRP, 2 * (int64_t)SLICE, KB, SLICE, CU_TENSOR_MAP_SWIZZLE_128B))) return rc;
  }
  if (op == nullptr) mop = mpre;              // unused by the launch: no main slices
  if (pre == nullptr) mpre = mmid = mop;      // unused by the launch: no expert GEMMs
  const int sms = sm_count();
  const int64_t n_tiles = (a.B + TM - 1) / TM;
  a.nsplit = in_place ? 1 : (int)std::max<int64_t>(1, std::min<int64_t>(sms / n_tiles, a.n_slices));
  const int KPmax = std::max(a.KP0, a.KRP);
  a.SB = std::min<int>(4, (int)((SMEM_CAP - 1024 - smem_bytes(KPmax, 0)) / (SBYTES + 16)));
  return launch(what, cross_mix_rows_wgmma_kernel, capped_grid(n_tiles * a.nsplit, sms), NTHREADS,
                smem_bytes(KPmax, a.SB) + 1024, st, mpre, mmid, mop, a);
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

extern "C" int ctr_cross_mix_workspace_bytes(int64_t B, int64_t d, int64_t L, int64_t K, int64_t r, int64_t* workspace_bytes,
                                             int64_t* saved_bytes) {
  static const char* fn = "ctr_cross_mix_workspace_bytes";
  CTR_REQUIRE(workspace_bytes != nullptr && saved_bytes != nullptr, "%s: null argument", fn);
  Shape s;
  if (int rc = shape_of(fn, B, d, L, K, r, s)) return rc;
  *workspace_bytes = s.bwd_bytes;
  *saved_bytes = s.saved_bytes;
  return CTR_OK;
}

extern "C" int ctr_cross_mix_fwd(const float* x0, const float* v, const float* c, const float* u, const float* b,
                                 const float* gate, int64_t B, int64_t d, int64_t L, int64_t K, int64_t r, int activation,
                                 float* out, void* saved, void* workspace, int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_cross_mix_fwd";
  Shape s;
  int rc = shape_of(fn, B, d, L, K, r, s);
  if (rc) return rc;
  CTR_REQUIRE(x0 && v && c && u && b && gate && out, "ctr_cross_mix_fwd: null argument");
  CTR_REQUIRE(activation == 0 || activation == 1, "%s: activation must be 1 (tanh) or 0 (identity), got %d", fn, activation);
  if ((rc = check_workspace(fn, "ctr_cross_mix_workspace_bytes with B = 0", workspace, workspace_bytes, s.weight_bytes)))
    return rc;
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  float* pre = static_cast<float*>(workspace);
  float* mid = pre + L * s.pre_floats;
  float* main = mid + L * s.mid_floats;
  if ((rc = prep("ctr_cross_mix_fwd(prep v)", OP_V, v, gate, pre, s.pre_floats, SLICE, s.DP, s, st)) ||
      (rc = prep("ctr_cross_mix_fwd(prep c)", OP_C, c, gate, mid, s.mid_floats, SLICE, s.KRP, s, st)) ||
      (rc = prep("ctr_cross_mix_fwd(prep u)", OP_U, u, gate, main, s.main_floats, s.NPd, s.KRP, s, st)))
    return rc;
  // saved: x_1 .. x_{L-1}, z_0 .. z_{L-1}, t_0 .. t_{L-1}, c~_0 .. c~_{L-1}, p_0 .. p_{L-1}
  float* xs = static_cast<float*>(saved);
  float* zs = xs == nullptr ? nullptr : xs + (L - 1) * B * d;
  float* ts = xs == nullptr ? nullptr : zs + L * B * d;
  float* cs = xs == nullptr ? nullptr : ts + L * B * s.KR;
  float* ps = xs == nullptr ? nullptr : cs + L * B * s.KR;
  for (int l = 0; l < s.L; ++l) {
    const float* xl = l == 0 ? x0 : (xs ? xs + (l - 1) * B * d : out);
    Args a = {};
    a.mode = FWD; a.act = activation;
    a.a = xl; a.lda = s.d; a.ka = s.d; a.KP0 = s.DP;
    a.K = s.K; a.r = s.r; a.KR = s.KR; a.KRP = s.KRP; a.gate = gate;
    a.t = ts ? ts + l * B * s.KR : nullptr;
    a.ct = cs ? cs + l * B * s.KR : nullptr;
    a.pg = ps ? ps + l * B * s.K : nullptr;
    a.KP = s.KRP; a.NP = s.NPd; a.n_slices = s.NPd / SLICE;
    a.epi = EPI_FWD; a.y = l == s.L - 1 || xs == nullptr ? out : xs + l * B * d;
    a.bias = b + (size_t)l * d; a.x0 = x0; a.xl = xl; a.z_out = zs ? zs + l * B * d : nullptr;
    a.B = (int)B; a.d = s.d;
    if ((rc = rows_gemm(fn, "ctr_cross_mix_fwd(wgmma)", a, pre + l * s.pre_floats, mid + l * s.mid_floats,
                        main + l * s.main_floats, xl == out, st)))
      return rc;
  }
  return CTR_OK;
}

extern "C" int ctr_cross_mix_bwd(const float* x0, const float* v, const float* c, const float* u, const float* b,
                                 const float* gate, const void* saved, const float* g_out, int64_t B, int64_t d, int64_t L,
                                 int64_t K, int64_t r, int activation, float* dx0, float* dv, float* dc, float* du, float* db,
                                 float* dgate, void* workspace, int64_t workspace_bytes, void* stream) {
  static const char* fn = "ctr_cross_mix_bwd";
  Shape s;
  int rc = shape_of(fn, B, d, L, K, r, s);
  if (rc) return rc;
  CTR_REQUIRE(x0 && v && c && u && b && gate && saved && g_out && dx0 && dv && dc && du && db && dgate,
              "ctr_cross_mix_bwd: null argument");
  CTR_REQUIRE(activation == 0 || activation == 1, "%s: activation must be 1 (tanh) or 0 (identity), got %d", fn, activation);
  if ((rc = check_workspace(fn, "ctr_cross_mix_workspace_bytes", workspace, workspace_bytes, s.bwd_bytes))) return rc;
  cudaStream_t st = as_stream(stream);
  const size_t per_layer = (size_t)s.KR * d;
  CTR_CUDA(cudaMemsetAsync(dv, 0, sizeof(float) * L * per_layer, st));
  CTR_CUDA(cudaMemsetAsync(du, 0, sizeof(float) * L * per_layer, st));
  CTR_CUDA(cudaMemsetAsync(dc, 0, sizeof(float) * (size_t)(L * K * r * r), st));
  CTR_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * (size_t)(L * d), st));
  CTR_CUDA(cudaMemsetAsync(dgate, 0, sizeof(float) * (size_t)(d * K), st));
  if (B == 0) return CTR_OK;
  float* S = at(workspace, s.s_off);
  CTR_CUDA(cudaMemsetAsync(S, 0, sizeof(float) * (size_t)(L * s.KR * s.KR), st));
  float* pre = static_cast<float*>(workspace);
  float* mid = pre + L * s.pre_floats;
  float* main = mid + L * s.mid_floats;
  if ((rc = prep("ctr_cross_mix_bwd(prep u)", OP_UT, u, gate, pre, s.pre_floats, SLICE, s.DP, s, st)) ||
      (rc = prep("ctr_cross_mix_bwd(prep c)", OP_CT, c, gate, mid, s.mid_floats, SLICE, s.KRP, s, st)) ||
      (rc = prep("ctr_cross_mix_bwd(prep v, gate)", OP_VG, v, gate, main, s.main_floats, s.NPd, s.W2, s, st)))
    return rc;
  float* xs = const_cast<float*>(static_cast<const float*>(saved));   // read only
  float* zs = xs + (L - 1) * B * d;
  float* ts = zs + L * B * d;
  float* cs = ts + L * B * s.KR;
  float* ps = cs + L * B * s.KR;
  float* dz = at(workspace, s.dz_off);
  float* aw = at(workspace, s.a_off);
  float* dm = at(workspace, s.dm_off);
  float* wq = at(workspace, s.w_off);
  const float* g = g_out;
  for (int l = s.L - 1; l >= 0; --l) {
    const float* xl = l == 0 ? x0 : xs + (l - 1) * B * d;
    float* gnext = l == 0 ? nullptr : at(workspace, s.g_off[(s.L - 1 - l) & 1]);
    float* tl = ts + l * B * s.KR;
    Args a = {};
    a.mode = BWD_CHAIN; a.act = activation;
    a.a = g; a.a_mul = x0; a.a_copy = dz; a.lda = s.d; a.ka = s.d; a.KP0 = s.DP;
    a.K = s.K; a.r = s.r; a.KR = s.KR; a.KRP = s.KRP;
    a.t = tl; a.ct = cs + l * B * s.KR; a.pg = ps + l * B * s.K;
    a.a_out = aw; a.dm_out = dm; a.w_out = wq; a.ldw = s.W2;
    a.B = (int)B; a.d = s.d;
    if ((rc = rows_gemm(fn, "ctr_cross_mix_bwd(experts, wgmma)", a, pre + l * s.pre_floats, mid + l * s.mid_floats, nullptr,
                        true, st)))
      return rc;
    a = Args{};
    a.mode = BWD_DX;
    a.a = wq; a.lda = s.W2; a.ka = s.KR + s.K; a.KP0 = s.W2;
    a.KP = s.W2; a.NP = s.NPd; a.n_slices = s.NPd / SLICE;
    a.epi = EPI_BWD; a.y = gnext; a.g = g; a.z = zs + l * B * d; a.x0 = x0; a.dx0 = dx0;
    a.dx0_accumulate = l < s.L - 1; a.dx0_add_dx = l == 0;
    a.B = (int)B; a.d = s.d;
    if ((rc = rows_gemm(fn, "ctr_cross_mix_bwd(dx, wgmma)", a, nullptr, nullptr, main + l * s.main_floats, false, st)))
      return rc;
    const Rows rdu = {du + l * per_layer, db + (size_t)l * d, s.d, s.d, 0, s.d, nullptr, 0, 0};
    const Rows rdv = {dv + l * per_layer, nullptr, s.KR, s.r, s.d * s.r, s.r, dgate, s.K, s.K};
    const Rows rdc = {S + (size_t)l * s.KR * s.KR, nullptr, s.KR, s.KR, 0, s.KR, nullptr, 0, 0};
    if ((rc = weight_grad(fn, "ctr_cross_mix_bwd(du, wgmma)", rdu, dz, s.DP, B, aw, s.KR, st)) ||
        (rc = weight_grad(fn, "ctr_cross_mix_bwd(dv, dgate, wgmma)", rdv, wq, s.W2, B, xl, s.d, st)) ||
        (rc = weight_grad(fn, "ctr_cross_mix_bwd(dc, wgmma)", rdc, dm, s.KRP, B, tl, s.KR, st)))
      return rc;
    g = gnext;
  }
  const int64_t n_dc = L * K * r * r;
  return launch("ctr_cross_mix_bwd(fold dc)", cross_mix_fold_kernel, capped_grid((n_dc + 255) / 256, 1024), 256, 0, st, S,
                dc, s.L, s.K, s.r);
}

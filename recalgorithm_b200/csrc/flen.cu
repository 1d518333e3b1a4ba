// FLEN field-wise bi-interaction (FwBI; Chen et al., arXiv:1911.04690): the fused per-field lookup and the layer that follows
// it.  The reference README lists FLEN as a to-do, so there is no reference code; the contract is the definition below,
// checked against a float64 restatement (tests/_flen_ref.py) and, through two degenerate groupings, against the NFM and FwFM
// fixtures executed from the reference's own lines.
//
// Fields are mapped to M <= 8 groups, group[f] in [0, M).  Per sample, with p_m = sum_{f in m} e_f and q_m = sum_{f in m} e_f^2
// (element-wise over D):
//   h = sum_{i<j} kernel_mf[pair(i,j)] p_i p_j + bias_mf  +  sum_m kernel_fm[m] (p_m^2 - q_m) + bias_fm        (B, D)
// pair(i,j): the row-major strict upper triangle of M x M (itertools.combinations order).  With g = dL/dh, for f in group m:
//   row_grads[b,f] = d_tile[b,f] + g (sum_{j != m} kernel_mf[pair(m,j)] p_j + 2 kernel_fm[m] (p_m - e_f))
//   d_kernel_mf[pair(i,j)] = sum_{b,d} g p_i p_j,  d_kernel_fm[m] = sum_{b,d} g (p_m^2 - q_m),  d_bias_mf = d_bias_fm = sum_b g.
//
// H100 mapping (HBM-bound gather, a few FLOPs per byte; no tensor cores), the FM2 lookup's (embed_fm2.cu): one warp per
// sample, a row of D fp32 is LPR = D/4 lanes x 128 bits, the ids of 32 fields are read with one coalesced load and shuffled
// so every row address is known before the first row load.  The group of a field is a run-time value, so the per-lane group
// sums p_m, q_m are register arrays updated by an unrolled select over NG compile-time slots (a dynamically indexed register
// array would live in local memory); NG = 4 serves M <= 4 (the paper's setting) with half the registers and select work of
// NG = 8.  The group map travels as a 256-byte kernel parameter.
// p_m^2 - q_m is squared then subtracted with no FMA contraction, so a singleton group gives exactly 0 (as the FM2 term does
// at F = 1), and so does its share of d_kernel_fm and of the row gradient.
#include "lookup_bwd.cuh"

namespace ctr {

constexpr int FWBI_MAX_GROUPS = 8;
constexpr int FWBI_MAX_FIELDS = 256;

struct FieldGroups {
  unsigned char g[FWBI_MAX_FIELDS];
};

__device__ __forceinline__ void f4_add(float4& a, const float4& v) { a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w; }
// a += v*v, squared then added (no contraction)
__device__ __forceinline__ void f4_add_sq(float4& a, const float4& v) {
  a.x = __fadd_rn(a.x, __fmul_rn(v.x, v.x)); a.y = __fadd_rn(a.y, __fmul_rn(v.y, v.y));
  a.z = __fadd_rn(a.z, __fmul_rn(v.z, v.z)); a.w = __fadd_rn(a.w, __fmul_rn(v.w, v.w));
}
// p*p - q, squared then subtracted (no contraction): exactly 0 for a singleton group
__device__ __forceinline__ float4 f4_sq_minus(const float4& p, const float4& q) {
  return make_float4(__fsub_rn(__fmul_rn(p.x, p.x), q.x), __fsub_rn(__fmul_rn(p.y, p.y), q.y),
                     __fsub_rn(__fmul_rn(p.z, p.z), q.z), __fsub_rn(__fmul_rn(p.w, p.w), q.w));
}
__device__ __forceinline__ float dot4(const float4& a, const float4& b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }

// p[grp] += v, q[grp] += v*v by select over the compile-time slots
template <int NG>
__device__ __forceinline__ void group_add(float4 (&p)[NG], float4 (&q)[NG], int grp, const float4& v) {
#pragma unroll
  for (int m = 0; m < NG; ++m)
    if (m == grp) { f4_add(p[m], v); f4_add_sq(q[m], v); }
}

// Forward.  TILE_IN: rows come from a (B, F, D) tile (row b*F + f); otherwise from the (V_total, D) table through
// row_off and ids (int64 or int32; OOV / out-of-range ids give zero rows), and the tile is written when given.  The weights
// and biases are read as floats: they need only float alignment.
// A floor of 2 CTAs per SM (at most 128 registers): with no floor, ptxas held the NG = 4 forms to 80 registers or fewer and
// spilled.
template <int LPR, int NG, typename IdT, bool TILE_IN>
__global__ void __launch_bounds__(256, 2)
fwbi_fwd_kernel(const float4* __restrict__ src, const long long* __restrict__ row_off, const IdT* __restrict__ ids, int B, int F,
                int M, const FieldGroups groups, const float* __restrict__ kmf, const float* __restrict__ kfm,
                const float* __restrict__ bmf, const float* __restrict__ bfm, float4* __restrict__ tile,
                float4* __restrict__ h, long long* __restrict__ ids64_out) {
  constexpr int RPW = 32 / LPR;
  constexpr int UB = LPR < 8 ? LPR : 8;
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR;
  const int c = lane % LPR;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;

  for (int b = warp0; b < B; b += nwarps) {
    float4 p[NG], q[NG];
#pragma unroll
    for (int m = 0; m < NG; ++m) { p[m] = f4_zero(); q[m] = f4_zero(); }
    for (int f0 = 0; f0 < F; f0 += 32) {
      const int nf = min(32, F - f0);
      long long row = -1;
      if (lane < nf) {
        if constexpr (TILE_IN) {
          row = (long long)b * F + f0 + lane;
        } else {
          const long long id = load_id(ids + (size_t)b * F + f0 + lane);
          const long long lo = __ldg(row_off + f0 + lane), hi = __ldg(row_off + f0 + lane + 1);
          row = (id >= 0 && id < hi - lo) ? lo + id : -1;
          if (sizeof(IdT) == 4 && ids64_out != nullptr) ids64_out[(size_t)b * F + f0 + lane] = id;
        }
      }
#pragma unroll
      for (int it0 = 0; it0 < LPR; it0 += UB) {
        if (it0 * RPW >= nf) break;                           // warp-uniform
        float4 v[UB];
        bool in[UB];
#pragma unroll
        for (int u = 0; u < UB; ++u) {
          const int fs = (it0 + u) * RPW + sub;
          const long long r = __shfl_sync(full, row, fs);
          in[u] = fs < nf;
          v[u] = f4_zero();
          if (in[u] && r >= 0) v[u] = ldg_stream_f4(src + (size_t)r * LPR + c);
        }
#pragma unroll
        for (int u = 0; u < UB; ++u) {
          if (!in[u]) continue;
          const int f = f0 + (it0 + u) * RPW + sub;
          group_add(p, q, groups.g[f], v[u]);
          if (!TILE_IN && tile != nullptr) stg_stream_f4(tile + ((size_t)b * F + f) * LPR + c, v[u]);
        }
      }
    }
#pragma unroll
    for (int m = 0; m < NG; ++m)
      if (m < M) { lane_group_sum<LPR>(p[m]); lane_group_sum<LPR>(q[m]); }   // M is warp-uniform
    if (lane < LPR) {
      float4 mf = make_float4(__ldg(bmf + 4 * c), __ldg(bmf + 4 * c + 1), __ldg(bmf + 4 * c + 2), __ldg(bmf + 4 * c + 3));
      float4 fm = make_float4(__ldg(bfm + 4 * c), __ldg(bfm + 4 * c + 1), __ldg(bfm + 4 * c + 2), __ldg(bfm + 4 * c + 3));
      int pr = 0;
#pragma unroll
      for (int i = 0; i < NG; ++i) {
        if (i >= M) break;
        const float4 t = f4_sq_minus(p[i], q[i]);
        const float k = __ldg(kfm + i);
        fm.x += k * t.x; fm.y += k * t.y; fm.z += k * t.z; fm.w += k * t.w;
#pragma unroll
        for (int j = i + 1; j < NG; ++j) {
          if (j >= M) break;
          const float w = __ldg(kmf + pr++);
          mf.x += w * (p[i].x * p[j].x); mf.y += w * (p[i].y * p[j].y);
          mf.z += w * (p[i].z * p[j].z); mf.w += w * (p[i].w * p[j].w);
        }
      }
      h[(size_t)b * LPR + c] = make_float4(mf.x + fm.x, mf.y + fm.y, mf.z + fm.z, mf.w + fm.w);
    }
  }
}

// Backward, from the tile (both forward forms).  One warp per sample: p_m, q_m from the tile row (held in registers with
// HOLD > 0, re-read in a second pass with HOLD == 0), then per group a_m = sum_{j != m} kernel_mf[pair(m,j)] p_j and
// s_m = 2 kernel_fm[m], then row_grads = d_tile + g (a_m + s_m (p_m - e)).  The weight-gradient partials of the lane's chunk
// are accumulated by the lanes < LPR only (after the lane-group sums every row slot holds the same p_m), reduced per CTA in
// shared memory and added to the (zeroed) outputs with one atomicAdd per element per CTA.
// Shared memory: [NG(NG-1)/2] d_kernel_mf, [NG] d_kernel_fm, [LPR] float4 d_bias.
template <int LPR, int HOLD, int NG>
__global__ void __launch_bounds__(256)
fwbi_bwd_kernel(const float4* __restrict__ tile, const float4* __restrict__ d_tile, const float4* __restrict__ d_h, int B, int F,
                int M, const FieldGroups groups, const float* __restrict__ kmf, const float* __restrict__ kfm,
                float4* __restrict__ row_grads, float* __restrict__ d_kmf, float* __restrict__ d_kfm, float* __restrict__ d_bmf,
                float* __restrict__ d_bfm) {
  constexpr int NP = NG * (NG - 1) / 2;
  __shared__ float s_kmf[NP], s_kfm[NG];
  __shared__ float4 s_b[LPR];
  for (int t = threadIdx.x; t < NP + NG + 4 * LPR; t += blockDim.x) {
    if (t < NP) s_kmf[t] = 0.f;
    else if (t < NP + NG) s_kfm[t - NP] = 0.f;
    else reinterpret_cast<float*>(s_b)[t - NP - NG] = 0.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int c = lane % LPR;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int n4 = F * LPR;
  // weight-gradient partials of this lane's chunk, indexed by the compile-time pair slot of (i, j) in the NG x NG triangle
  float acc_mf[NP], acc_fm[NG];
  float4 acc_b = f4_zero();
#pragma unroll
  for (int k = 0; k < NP; ++k) acc_mf[k] = 0.f;
#pragma unroll
  for (int k = 0; k < NG; ++k) acc_fm[k] = 0.f;

  for (int b = warp0; b < B; b += nwarps) {
    const float4* e_row = tile + (size_t)b * n4;
    const float4 g = __ldg(d_h + (size_t)b * LPR + c);
    float4 p[NG], q[NG];
#pragma unroll
    for (int m = 0; m < NG; ++m) { p[m] = f4_zero(); q[m] = f4_zero(); }
    float4 e[HOLD > 0 ? HOLD : 1], dt[HOLD > 0 ? HOLD : 1];
    if constexpr (HOLD > 0) {
      load_tile_row(e, e_row, n4, lane, [](int, int) {});
#pragma unroll
      for (int k = 0; k < HOLD; ++k) {
        const int j = k * 32 + lane;
        dt[k] = f4_zero();
        if (j < n4) {
          if (d_tile != nullptr) dt[k] = ldg_stream_f4(d_tile + (size_t)b * n4 + j);
          group_add(p, q, groups.g[j / LPR], e[k]);
        }
      }
    } else {
      for (int j = lane; j < n4; j += 32) group_add(p, q, groups.g[j / LPR], __ldg(e_row + j));
    }
#pragma unroll
    for (int m = 0; m < NG; ++m)
      if (m < M) { lane_group_sum<LPR>(p[m]); lane_group_sum<LPR>(q[m]); }   // M is warp-uniform
    if (lane < LPR) {                 // one count per chunk, not one per row slot
      f4_add(acc_b, g);
#pragma unroll
      for (int i = 0, k = 0; i < NG; ++i) {
        acc_fm[i] += dot4(g, f4_sq_minus(p[i], q[i]));
#pragma unroll
        for (int j = i + 1; j < NG; ++j, ++k)
          acc_mf[k] += dot4(g, make_float4(p[i].x * p[j].x, p[i].y * p[j].y, p[i].z * p[j].z, p[i].w * p[j].w));
      }
    }
    // per-group coefficient vectors; q is dead from here on, a_m takes its registers
    float4 a[NG];
    float s[NG];
#pragma unroll
    for (int m = 0; m < NG; ++m) { a[m] = f4_zero(); s[m] = m < M ? 2.f * __ldg(kfm + m) : 0.f; }
    {
      int pr = 0;
#pragma unroll
      for (int i = 0; i < NG; ++i) {
        if (i >= M) break;
#pragma unroll
        for (int j = i + 1; j < NG; ++j) {
          if (j >= M) break;
          const float w = __ldg(kmf + pr++);
          a[i].x += w * p[j].x; a[i].y += w * p[j].y; a[i].z += w * p[j].z; a[i].w += w * p[j].w;
          a[j].x += w * p[i].x; a[j].y += w * p[i].y; a[j].z += w * p[i].z; a[j].w += w * p[i].w;
        }
      }
    }
    auto row_grad = [&](int j, const float4& v, const float4& d) {
      const int grp = groups.g[j / LPR];
      float4 am = a[0], pm = p[0];
      float sm = s[0];
#pragma unroll
      for (int m = 1; m < NG; ++m)
        if (m == grp) { am = a[m]; pm = p[m]; sm = s[m]; }
      float4 r;
      r.x = d.x + g.x * (am.x + sm * (pm.x - v.x)); r.y = d.y + g.y * (am.y + sm * (pm.y - v.y));
      r.z = d.z + g.z * (am.z + sm * (pm.z - v.z)); r.w = d.w + g.w * (am.w + sm * (pm.w - v.w));
      stg_stream_f4(row_grads + (size_t)b * n4 + j, r);
    };
    if constexpr (HOLD > 0) {
#pragma unroll
      for (int k = 0; k < HOLD; ++k) {
        const int j = k * 32 + lane;
        if (j < n4) row_grad(j, e[k], dt[k]);
      }
    } else {
      for (int j = lane; j < n4; j += 32) {
        const float4 d = d_tile != nullptr ? ldg_stream_f4(d_tile + (size_t)b * n4 + j) : f4_zero();
        row_grad(j, __ldg(e_row + j), d);
      }
    }
  }
  // per-CTA reduction: the LPR lanes of a warp sum their scalar partials, lane 0 adds them to shared memory
#pragma unroll
  for (int k = 0; k < NP; ++k)
#pragma unroll
    for (int o = 1; o < LPR; o <<= 1) acc_mf[k] += __shfl_xor_sync(0xffffffffu, acc_mf[k], o);
#pragma unroll
  for (int k = 0; k < NG; ++k)
#pragma unroll
    for (int o = 1; o < LPR; o <<= 1) acc_fm[k] += __shfl_xor_sync(0xffffffffu, acc_fm[k], o);
  if (lane == 0) {
    int pr = 0;
#pragma unroll
    for (int i = 0, k = 0; i < NG; ++i) {
      if (i < M) atomicAdd(s_kfm + i, acc_fm[i]);
#pragma unroll
      for (int j = i + 1; j < NG; ++j, ++k)
        if (j < M) atomicAdd(s_kmf + pr++, acc_mf[k]);
    }
  }
  if (lane < LPR) {
    float* sb = reinterpret_cast<float*>(s_b + c);
    atomicAdd(sb + 0, acc_b.x); atomicAdd(sb + 1, acc_b.y); atomicAdd(sb + 2, acc_b.z); atomicAdd(sb + 3, acc_b.w);
  }
  __syncthreads();
  const int np = M * (M - 1) / 2;
  for (int t = threadIdx.x; t < np + M + 4 * LPR; t += blockDim.x) {
    if (t < np) {
      atomicAdd(d_kmf + t, s_kmf[t]);
    } else if (t < np + M) {
      atomicAdd(d_kfm + t - np, s_kfm[t - np]);
    } else {
      const float v = reinterpret_cast<const float*>(s_b)[t - np - M];
      atomicAdd(d_bmf + t - np - M, v);
      atomicAdd(d_bfm + t - np - M, v);
    }
  }
}

// The slot count of a kernel for M groups
template <class Fn>
int with_slots(int64_t M, Fn&& f) {
  if (M <= 4) return f(std::integral_constant<int, 4>{});
  return f(std::integral_constant<int, FWBI_MAX_GROUPS>{});
}

// Checks what every FwBI entry shares: the (B, F, D) bounds of the row kernels, F <= 256, 1 <= M <= 8, the host group map
// (each entry in [0, M)) and the weights (kernel_mf may be NULL only when M == 1); fills the kernel's group parameter.
static int check_fwbi(const char* fn, int64_t B, int64_t F, int64_t D, const int32_t* field_group, int64_t M, const float* kmf,
                      const float* kfm, FieldGroups& groups) {
  int rc = check_bfd(fn, B, F, D);
  if (rc) return rc;
  CTR_UNSUPPORTED(F > FWBI_MAX_FIELDS, "%s: F=%lld fields exceed the bound F <= %d", fn, (long long)F, FWBI_MAX_FIELDS);
  CTR_UNSUPPORTED(M < 1 || M > FWBI_MAX_GROUPS, "%s: M=%lld groups outside the bound 1 <= M <= %d", fn, (long long)M,
                  FWBI_MAX_GROUPS);
  CTR_REQUIRE(field_group && kfm && (kmf || M == 1), "%s: null field_group/kernel_mf/kernel_fm", fn);
  for (int64_t f = 0; f < F; ++f) {
    CTR_REQUIRE(field_group[f] >= 0 && field_group[f] < M, "%s: field_group[%lld]=%d outside [0, M=%lld)", fn, (long long)f,
                (int)field_group[f], (long long)M);
    groups.g[f] = (unsigned char)field_group[f];
  }
  for (int64_t f = F; f < FWBI_MAX_FIELDS; ++f) groups.g[f] = 0;
  return CTR_OK;
}

template <typename IdT, bool TILE_IN>
static int launch_fwbi_fwd(const char* fn, const float* src, const int64_t* off, const IdT* ids, int64_t B, int64_t F, int64_t D,
                           int64_t M, const FieldGroups& groups, const float* kmf, const float* kfm, const float* bmf,
                           const float* bfm, float* tile, float* h, int64_t* ids64_out, cudaStream_t st) {
  return with_lpr(D, [&](auto LPR) {
    return with_slots(M, [&](auto NG) {
      return launch_resident(fn, fwbi_fwd_kernel<LPR, NG, IdT, TILE_IN>, (B + 7) / 8, 256, 0, st,
                             reinterpret_cast<const float4*>(src), reinterpret_cast<const long long*>(off), ids, (int)B, (int)F,
                             (int)M, groups, kmf, kfm, bmf, bfm, reinterpret_cast<float4*>(tile), reinterpret_cast<float4*>(h),
                             reinterpret_cast<long long*>(ids64_out));
    });
  });
}

}  // namespace ctr

using namespace ctr;

extern "C" int ctr_embed_fwbi_fwd(const float* table, const int64_t* field_row_offset, const void* ids, int ids_are_int32,
                                  int64_t B, int64_t F, int64_t D, const int32_t* field_group, int64_t M,
                                  const float* kernel_mf, const float* kernel_fm, const float* bias_mf, const float* bias_fm,
                                  float* tile, float* h, int64_t* ids64_out, void* stream) {
  const char* fn = "ctr_embed_fwbi_fwd";
  FieldGroups groups;
  int rc = check_fwbi(fn, B, F, D, field_group, M, kernel_mf, kernel_fm, groups);
  if (rc) return rc;
  CTR_REQUIRE(table && field_row_offset && ids && bias_mf && bias_fm && h,
              "%s: null table/field_row_offset/ids/bias_mf/bias_fm/h", fn);
  CTR_REQUIRE(aligned16(table) && aligned16(tile) && aligned16(h), "%s: table, tile and h must be 16-byte aligned", fn);
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  if (ids_are_int32)
    return launch_fwbi_fwd<int, false>(fn, table, field_row_offset, reinterpret_cast<const int*>(ids), B, F, D, M, groups,
                                       kernel_mf, kernel_fm, bias_mf, bias_fm, tile, h, ids64_out, st);
  return launch_fwbi_fwd<long long, false>(fn, table, field_row_offset, reinterpret_cast<const long long*>(ids), B, F, D, M,
                                           groups, kernel_mf, kernel_fm, bias_mf, bias_fm, tile, h, nullptr, st);
}

extern "C" int ctr_fwbi_fwd(const float* tile, int64_t B, int64_t F, int64_t D, const int32_t* field_group, int64_t M,
                            const float* kernel_mf, const float* kernel_fm, const float* bias_mf, const float* bias_fm, float* h,
                            void* stream) {
  const char* fn = "ctr_fwbi_fwd";
  FieldGroups groups;
  int rc = check_fwbi(fn, B, F, D, field_group, M, kernel_mf, kernel_fm, groups);
  if (rc) return rc;
  CTR_REQUIRE(tile && bias_mf && bias_fm && h, "%s: null tile/bias_mf/bias_fm/h", fn);
  CTR_REQUIRE(aligned16(tile) && aligned16(h), "%s: tile and h must be 16-byte aligned", fn);
  if (B == 0) return CTR_OK;
  return launch_fwbi_fwd<long long, true>(fn, tile, nullptr, nullptr, B, F, D, M, groups, kernel_mf, kernel_fm, bias_mf, bias_fm,
                                          nullptr, h, nullptr, as_stream(stream));
}

extern "C" int ctr_fwbi_bwd(const float* tile, const float* d_tile, const float* d_h, int64_t B, int64_t F, int64_t D,
                            const int32_t* field_group, int64_t M, const float* kernel_mf, const float* kernel_fm,
                            float* row_grads, float* d_kernel_mf, float* d_kernel_fm, float* d_bias_mf, float* d_bias_fm,
                            void* stream) {
  const char* fn = "ctr_fwbi_bwd";
  FieldGroups groups;
  int rc = check_fwbi(fn, B, F, D, field_group, M, kernel_mf, kernel_fm, groups);
  if (rc) return rc;
  CTR_REQUIRE(tile && d_h && row_grads && (d_kernel_mf || M == 1) && d_kernel_fm && d_bias_mf && d_bias_fm,
              "%s: null tile/d_h/row_grads/d_kernel_mf/d_kernel_fm/d_bias_mf/d_bias_fm", fn);
  CTR_REQUIRE(aligned16(tile) && aligned16(d_tile) && aligned16(d_h) && aligned16(row_grads),
              "%s: tile, d_tile, d_h and row_grads must be 16-byte aligned", fn);
  cudaStream_t st = as_stream(stream);
  if (M > 1) CTR_CUDA(cudaMemsetAsync(d_kernel_mf, 0, sizeof(float) * (M * (M - 1) / 2), st));
  CTR_CUDA(cudaMemsetAsync(d_kernel_fm, 0, sizeof(float) * M, st));
  CTR_CUDA(cudaMemsetAsync(d_bias_mf, 0, sizeof(float) * D, st));
  CTR_CUDA(cudaMemsetAsync(d_bias_fm, 0, sizeof(float) * D, st));
  if (B == 0) return CTR_OK;
  return with_lpr(D, [&](auto LPR) {
    return with_hold<true>(F, LPR, [&](auto HOLD) {
      return with_slots(M, [&](auto NG) {
        return launch_resident(fn, fwbi_bwd_kernel<LPR, HOLD, NG>, (B + 7) / 8, 256, 0, st, reinterpret_cast<const float4*>(tile),
                               reinterpret_cast<const float4*>(d_tile), reinterpret_cast<const float4*>(d_h), (int)B, (int)F,
                               (int)M, groups, kernel_mf, kernel_fm, reinterpret_cast<float4*>(row_grads), d_kernel_mf,
                               d_kernel_fm, d_bias_mf, d_bias_fm);
      });
    }, fn);
  });
}

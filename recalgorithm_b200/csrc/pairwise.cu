// SURVEY.md 8f.4 -- pairwise siblings of FM2 that consume the (B, F, K) tile of the lookup:
//
//   FwFM  (FwFM/fwfm.py:140-158)  logit[b] = sum_{i<j} r[pair(i,j)] * <e_i, e_j>,   pair() = utils.py:67-82 (row-major
//                                  strict upper triangle)
//   AFM   (AFM/afm.py:152-186)    had_p = e_i * e_j (i<j);  a_p = h^T relu(W^T had_p + b);  s = softmax_p(a);
//                                  pooled[b,:] = sum_p s_p * had_p          (the (B,P,K) tensor is never materialised)
//
// Both are CUDA-core kernels, one warp per sample, the sample's F x K block staged in shared memory.  AFM follows the DIN
// attention layout: lane u owns hidden unit(s) u, u+32, ... of the attention MLP with its W column and (backward) dW
// column in registers for the whole kernel; per pair the hadamard vector is a shared-memory broadcast.
#include "ctr_common.cuh"

namespace ctr {

constexpr int PW_WARPS = 4;

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------------------------- FwFM
// smem: R (F x F, symmetric, zero diagonal) | BWD: d_r accumulator (P) | per warp: e (F x KP)
// VEC (K % 4 == 0): rows padded to KP = K + 4 floats, every shared load is 128-bit (eight consecutive rows start in eight
// different banks); one pair per lane; the backward's R * E product computes four adjacent k per thread.
template <bool BWD, bool VEC>
__global__ void __launch_bounds__(PW_WARPS * 32)
fwfm_kernel(const float* __restrict__ tile, const float* __restrict__ r, const float* __restrict__ g, int B, int F, int K,
            float* __restrict__ out, float* __restrict__ d_tile, float* __restrict__ d_r) {
  extern __shared__ __align__(16) float sm[];
  const int KP = VEC ? K + 4 : K + 1, P = F * (F - 1) / 2, PP = (P + 3) & ~3, FF = (F * F + 3) & ~3;
  float* Rs = sm;                                   // F*F
  float* drs = Rs + FF;                             // BWD: P   (CTA-level accumulator of d_r)
  float* es = drs + (BWD ? PP : 0) + (threadIdx.x >> 5) * F * KP;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int x = threadIdx.x; x < F * F; x += blockDim.x) {
    const int i = x / F, j = x % F;
    const int lo = i < j ? i : j, hi = i < j ? j : i;
    Rs[x] = (i == j) ? 0.f : __ldg(r + lo * (F - 1) - lo * (lo - 1) / 2 + (hi - lo - 1));
  }
  if (BWD)
    for (int x = threadIdx.x; x < P; x += blockDim.x) drs[x] = 0.f;
  __syncthreads();

  for (int b = blockIdx.x * PW_WARPS + warp; b < B; b += gridDim.x * PW_WARPS) {
    const float* src = tile + (size_t)b * F * K;
    for (int x = lane; x < F * K; x += 32) es[(x / K) * KP + x % K] = __ldg(src + x);
    __syncwarp();
    const float gb = BWD ? __ldg(g + b) : 0.f;
    // pair-per-lane: p = lane, lane+32, ... in the reference's pair order; (i, j) advanced incrementally (row i holds F-1-i pairs)
    float acc = 0.f;
    int i = 0, j = 1 + lane;
    while (i < F - 1 && j >= F) { j = j - F + i + 2; ++i; }
    for (int p = lane; p < P; p += 32) {
      const float* ei = es + i * KP;
      const float* ej = es + j * KP;
      float dot = 0.f;
      if (VEC) {
        for (int k = 0; k < K; k += 4) {
          const float4 a = *reinterpret_cast<const float4*>(ei + k), c = *reinterpret_cast<const float4*>(ej + k);
          dot = fmaf(a.x, c.x, dot); dot = fmaf(a.y, c.y, dot); dot = fmaf(a.z, c.z, dot); dot = fmaf(a.w, c.w, dot);
        }
      } else {
        for (int k = 0; k < K; ++k) dot = fmaf(ei[k], ej[k], dot);
      }
      if (BWD) atomicAdd(drs + p, gb * dot); else acc = fmaf(Rs[i * F + j], dot, acc);
      j += 32;
      while (i < F - 1 && j >= F) { j = j - F + i + 2; ++i; }
    }
    if (!BWD) {
      acc = warp_sum(acc);
      if (lane == 0) out[b] = acc;
    } else {
      // d e_i[k] = g * sum_j R[i][j] e_j[k]
      float* dst = d_tile + (size_t)b * F * K;
      if (VEC) {
        const int K4 = K >> 2;
        for (int x = lane; x < F * K4; x += 32) {
          const int ii = x / K4, k = (x - ii * K4) * 4;
          float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int jj = 0; jj < F; ++jj) {
            const float rij = Rs[ii * F + jj];
            const float4 c = *reinterpret_cast<const float4*>(es + jj * KP + k);
            s4.x = fmaf(rij, c.x, s4.x); s4.y = fmaf(rij, c.y, s4.y); s4.z = fmaf(rij, c.z, s4.z); s4.w = fmaf(rij, c.w, s4.w);
          }
          *reinterpret_cast<float4*>(dst + ii * K + k) = make_float4(gb * s4.x, gb * s4.y, gb * s4.z, gb * s4.w);
        }
      } else {
        for (int x = lane; x < F * K; x += 32) {
          const int ii = x / K, k = x % K;
          float s1 = 0.f;
          for (int jj = 0; jj < F; ++jj) s1 = fmaf(Rs[ii * F + jj], es[jj * KP + k], s1);
          dst[x] = gb * s1;
        }
      }
    }
    __syncwarp();
  }
  if (BWD) {
    __syncthreads();
    for (int x = threadIdx.x; x < P; x += blockDim.x) atomicAdd(d_r + x, drs[x]);
  }
}

// -------------------------------------------------------------------------------------------------------------- AFM
// all-lane total of v[lane & (K-1)] (xor stages for offsets >= K, then a halving butterfly: K-1 shuffles instead of 5K)
template <int K>
__device__ __forceinline__ float reduce_to_owner(float (&v)[K], int lane) {
  const unsigned full = 0xffffffffu;
#pragma unroll
  for (int o = 16; o >= K; o >>= 1)
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] += __shfl_xor_sync(full, v[k], o);
#pragma unroll
  for (int o = K / 2; o >= 1; o >>= 1) {
    const bool up = (lane & o) != 0;
#pragma unroll
    for (int x = 0; x < o; ++x) {
      const float send = up ? v[x] : v[x + o];
      const float keep = up ? v[x + o] : v[x];
      v[x] = keep + __shfl_xor_sync(full, send, o);
    }
  }
  return v[0];
}

// per-warp smem: es (F*K) | att (P) | BWD: ds (P) | des (F*K)
template <int K, int TU, bool BWD>
__global__ void __launch_bounds__(PW_WARPS * 32)
afm_kernel(const float* __restrict__ tile, const float* __restrict__ w, const float* __restrict__ bias,
           const float* __restrict__ hvec, const float* __restrict__ g_out, int B, int F, int T,
           float* __restrict__ pooled, float* __restrict__ score, float* __restrict__ d_tile, float* __restrict__ d_w,
           float* __restrict__ d_b, float* __restrict__ d_h) {
  extern __shared__ float sm[];
  const int P = F * (F - 1) / 2, FK = F * K, PP = (P + 3) & ~3;     // PP keeps every sub-array 16-byte aligned
  const int per_warp = FK + PP + (BWD ? PP + FK : 0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* es = sm + warp * per_warp;
  float* att = es + FK;
  float* ds = att + PP;          // BWD only
  float* des = ds + PP;          // BWD only
  const unsigned full = 0xffffffffu;

  float W[K][TU], bu[TU], hu[TU];
#pragma unroll
  for (int tu = 0; tu < TU; ++tu) {
    const int u = lane + 32 * tu;
    bu[tu] = u < T ? __ldg(bias + u) : 0.f;
    hu[tu] = u < T ? __ldg(hvec + u) : 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) W[k][tu] = u < T ? __ldg(w + k * T + u) : 0.f;
  }
  float dW[BWD ? K : 1][TU], dbu[TU], dhu[TU];
  if (BWD) {
#pragma unroll
    for (int tu = 0; tu < TU; ++tu) {
      dbu[tu] = 0.f; dhu[tu] = 0.f;
#pragma unroll
      for (int k = 0; k < (BWD ? K : 1); ++k) dW[k][tu] = 0.f;
    }
  }

  for (int b = blockIdx.x * PW_WARPS + warp; b < B; b += gridDim.x * PW_WARPS) {
    const float* src = tile + (size_t)b * FK;
    for (int x = lane; x < FK; x += 32) { es[x] = __ldg(src + x); if (BWD) des[x] = 0.f; }
    __syncwarp();
    // ---- pass 1: attention logits a_p
    int p = 0;
    for (int i = 0; i < F - 1; ++i)
      for (int j = i + 1; j < F; ++j, ++p) {
        float h[K];
#pragma unroll
        for (int k4 = 0; k4 < K; k4 += 4) {
          const float4 a = *reinterpret_cast<const float4*>(es + i * K + k4), c = *reinterpret_cast<const float4*>(es + j * K + k4);
          h[k4] = a.x * c.x; h[k4 + 1] = a.y * c.y; h[k4 + 2] = a.z * c.z; h[k4 + 3] = a.w * c.w;
        }
        float a = 0.f;
#pragma unroll
        for (int tu = 0; tu < TU; ++tu) {
          float pre = bu[tu];
#pragma unroll
          for (int k = 0; k < K; ++k) pre = fmaf(h[k], W[k][tu], pre);
          a = fmaf(hu[tu], fmaxf(pre, 0.f), a);
        }
        a = warp_sum(a);
        if (lane == 0) att[p] = a;
      }
    __syncwarp();
    // ---- softmax over the pair axis
    float mx = -INFINITY;
    for (int q = lane; q < P; q += 32) mx = fmaxf(mx, att[q]);
    mx = warp_max(mx);
    float den = 0.f;
    for (int q = lane; q < P; q += 32) { const float ex = expf(att[q] - mx); att[q] = ex; den += ex; }
    den = warp_sum(den);
    const float inv = 1.f / den;
    for (int q = lane; q < P; q += 32) {
      const float s = att[q] * inv;
      att[q] = s;
      if (!BWD && score != nullptr) score[(size_t)b * P + q] = s;
    }
    __syncwarp();
    const int kk = lane & (K - 1), grp = lane / K;         // K <= 32: 32/K pair groups
    constexpr int NG = 32 / K;
    if (!BWD) {
      // ---- pooled[k] = sum_p s_p * e_i[k] * e_j[k]
      float acc = 0.f;
      p = 0;
      for (int i = 0; i < F - 1; ++i)
        for (int j = i + 1; j < F; ++j, ++p)
          if (p % NG == grp) acc = fmaf(att[p], es[i * K + kk] * es[j * K + kk], acc);
#pragma unroll
      for (int o = 16; o >= K; o >>= 1) acc += __shfl_xor_sync(full, acc, o);
      if (lane < K) pooled[(size_t)b * K + lane] = acc;
    } else {
      const float gk = __ldg(g_out + (size_t)b * K + kk);
      // ---- pass 2: ds_p = <g, had_p> (lanes split k, butterfly over the K lanes of a group),  c = sum_p s_p ds_p
      float c = 0.f;
      p = 0;
      for (int i = 0; i < F - 1; ++i)
        for (int j = i + 1; j < F; ++j, ++p) {
          float v = gk * es[i * K + kk] * es[j * K + kk];
#pragma unroll
          for (int o = K / 2; o >= 1; o >>= 1) v += __shfl_xor_sync(full, v, o);     // all-lane: every group computes it
          if (lane == 0) ds[p] = v;
          if ((p & 31) == lane) c = fmaf(att[p], v, c);        // lane-strided partial sums + tree: c feeds every datt
        }
      c = warp_sum(c);
      __syncwarp();
      // ---- pass 3: per pair, backward through softmax, the MLP and the hadamard product
      p = 0;
      for (int i = 0; i < F - 1; ++i)
        for (int j = i + 1; j < F; ++j, ++p) {
          const float s = att[p], datt = s * (ds[p] - c);
          float h[K], part[K];
#pragma unroll
          for (int k4 = 0; k4 < K; k4 += 4) {
            const float4 a = *reinterpret_cast<const float4*>(es + i * K + k4), cc = *reinterpret_cast<const float4*>(es + j * K + k4);
            h[k4] = a.x * cc.x; h[k4 + 1] = a.y * cc.y; h[k4 + 2] = a.z * cc.z; h[k4 + 3] = a.w * cc.w;
          }
#pragma unroll
          for (int k = 0; k < K; ++k) part[k] = 0.f;
#pragma unroll
          for (int tu = 0; tu < TU; ++tu) {
            float pre = bu[tu];
#pragma unroll
            for (int k = 0; k < K; ++k) pre = fmaf(h[k], W[k][tu], pre);
            dhu[tu] = fmaf(fmaxf(pre, 0.f), datt, dhu[tu]);
            const float dpre = pre > 0.f ? datt * hu[tu] : 0.f;
            dbu[tu] += dpre;
#pragma unroll
            for (int k = 0; k < K; ++k) {
              dW[BWD ? k : 0][tu] = fmaf(h[k], dpre, dW[BWD ? k : 0][tu]);
              part[k] = fmaf(W[k][tu], dpre, part[k]);
            }
          }
          const float tot = reduce_to_owner<K>(part, lane);            // sum over hidden units, for k = lane & (K-1)
          if (lane < K) {
            const float dhad = fmaf(gk, s, tot);
            const float ei = es[i * K + lane], ej = es[j * K + lane];
            des[i * K + lane] = fmaf(dhad, ej, des[i * K + lane]);
            des[j * K + lane] = fmaf(dhad, ei, des[j * K + lane]);
          }
        }
      __syncwarp();
      float* dst = d_tile + (size_t)b * FK;
      for (int x = lane; x < FK; x += 32) dst[x] = des[x];
    }
    __syncwarp();
  }
  if (BWD) {
#pragma unroll
    for (int tu = 0; tu < TU; ++tu) {
      const int u = lane + 32 * tu;
      if (u < T) {
        atomicAdd(d_b + u, dbu[tu]);
        atomicAdd(d_h + u, dhu[tu]);
#pragma unroll
        for (int k = 0; k < K; ++k) atomicAdd(d_w + k * T + u, dW[BWD ? k : 0][tu]);
      }
    }
  }
}

// -------------------------------------------------------------------------------------------------------------- FFM
// Field-aware FM (FFM/ffm.py:128-160).  tile (B, F, F-1, K): field i keeps one sub-embedding per other field; slot s of field i
// faces field j = s + 1 (s >= i) or s (s < i), which faces i through slot i - 1 (i > j) or i.  Every (field, slot) position
// belongs to exactly one pair, so   out[b] = 0.5 * sum_{i,s,k} tile[b,i,s,k] * tile[b,partner(i,s),k]   and the backward is a
// permutation scaled by g: both are streaming element-wise kernels (one warp per sample, lanes over (i,s,k)).
__device__ __forceinline__ int ffm_partner_elem(int e, int F, int K) {
  const int k = e % K, is = e / K, s = is % (F - 1), i = is / (F - 1);
  const int j = s >= i ? s + 1 : s, sb = i > j ? i - 1 : i;
  return (j * (F - 1) + sb) * K + k;
}

template <bool BWD>
__global__ void __launch_bounds__(256)
ffm_kernel(const float* __restrict__ tile, const float* __restrict__ g, int B, int F, int K, float* __restrict__ out,
           float* __restrict__ d_tile) {
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const int n = F * (F - 1) * K;
  for (int b = warp0; b < B; b += nwarps) {
    const float* row = tile + (size_t)b * n;
    if (BWD) {
      const float gb = __ldg(g + b);
      for (int e = lane; e < n; e += 32) d_tile[(size_t)b * n + e] = gb * __ldg(row + ffm_partner_elem(e, F, K));
    } else {
      float acc = 0.f;
      for (int e = lane; e < n; e += 32) acc = fmaf(__ldg(row + e), __ldg(row + ffm_partner_elem(e, F, K)), acc);
      acc = warp_sum(acc);
      if (lane == 0) out[b] = 0.5f * acc;
    }
  }
}

template <int K, int TU, bool BWD>
static int afm_launch(const float* tile, const float* w, const float* b, const float* h, const float* g, int64_t B, int64_t F,
                      int64_t T, float* pooled, float* score, float* d_tile, float* d_w, float* d_b, float* d_h, cudaStream_t st) {
  const int64_t PP = (F * (F - 1) / 2 + 3) & ~3LL;
  const size_t smem = (size_t)PW_WARPS * (F * K + PP + (BWD ? PP + F * K : 0)) * sizeof(float);
  CTR_UNSUPPORTED(smem > 200 * 1024, "ctr_afm: F=%lld K=%d needs %zu bytes of shared memory", (long long)F, K, smem);
  return launch_resident(BWD ? "ctr_afm_bwd" : "ctr_afm_fwd", afm_kernel<K, TU, BWD>, (B + PW_WARPS - 1) / PW_WARPS, PW_WARPS * 32,
                         smem, st, tile, w, b, h, g, (int)B, (int)F, (int)T, pooled, score, d_tile, d_w, d_b, d_h);
}

template <bool BWD>
static int afm_dispatch(const float* tile, const float* w, const float* b, const float* h, const float* g, int64_t B, int64_t F,
                        int64_t K, int64_t T, float* pooled, float* score, float* d_tile, float* d_w, float* d_b, float* d_h,
                        cudaStream_t st) {
  const int64_t tu = (T + 31) / 32;
  // register budget: W (and dW in the backward) columns live in registers, K * TU <= 64 floats each
  CTR_UNSUPPORTED((K != 4 && K != 8 && K != 16 && K != 32) || tu > 8 || K * tu > 64,
                  "ctr_afm: K=%lld, attention_factor=%lld unsupported (K in {4,8,16,32}, K*ceil(t/32) <= 64)", (long long)K,
                  (long long)T);
  return with_const<4, 8, 16, 32>((int)K, [&](auto KK) {
    return with_const<1, 2, 4, 8>(tu <= 1 ? 1 : tu <= 2 ? 2 : tu <= 4 ? 4 : 8, [&](auto TU) {
      if constexpr (KK * TU <= 64) return afm_launch<KK, TU, BWD>(tile, w, b, h, g, B, F, T, pooled, score, d_tile, d_w, d_b, d_h, st);
      else return (int)CTR_ERR_UNSUPPORTED;   // refused above
    });
  });
}

}  // namespace ctr

using namespace ctr;

static int check_pw(const char* fn, int64_t B, int64_t F, int64_t K) {
  CTR_REQUIRE(B >= 0 && F >= 2 && K >= 1, "%s: bad sizes B=%lld F=%lld K=%lld (F >= 2)", fn, (long long)B, (long long)F, (long long)K);
  CTR_REQUIRE(B <= 0x7fffffffLL / 8 && F <= 1024, "%s: B=%lld / F=%lld too large", fn, (long long)B, (long long)F);
  return CTR_OK;
}

template <bool BWD, bool VEC>
static int fwfm_launch(const char* fn, const float* tile, const float* r, const float* g, int64_t B, int64_t F, int64_t K, float* out,
                       float* d_tile, float* d_r, cudaStream_t st) {
  const int64_t P = F * (F - 1) / 2, PP = (P + 3) & ~3LL, FF = (F * F + 3) & ~3LL, KP = VEC ? K + 4 : K + 1;
  const size_t smem = (size_t)(FF + (BWD ? PP : 0) + PW_WARPS * F * KP) * sizeof(float);
  CTR_UNSUPPORTED(smem > 200 * 1024, "%s: F=%lld K=%lld needs %zu bytes of shared memory", fn, (long long)F, (long long)K, smem);
  return launch_resident(fn, fwfm_kernel<BWD, VEC>, (B + PW_WARPS - 1) / PW_WARPS, PW_WARPS * 32, smem, st, tile, r, g, (int)B, (int)F,
                         (int)K, out, d_tile, d_r);
}

static int fwfm_run(bool bwd, const float* tile, const float* r, const float* g, int64_t B, int64_t F, int64_t K, float* out,
                    float* d_tile, float* d_r, void* stream) {
  const char* fn = bwd ? "ctr_fwfm_bwd" : "ctr_fwfm_fwd";
  int rc = check_pw(fn, B, F, K);
  if (rc) return rc;
  cudaStream_t st = as_stream(stream);
  if (bwd) CTR_CUDA(cudaMemsetAsync(d_r, 0, (size_t)(F * (F - 1) / 2) * sizeof(float), st));
  if (B == 0) return CTR_OK;
  // 128-bit path: K a multiple of 4 and 16-byte aligned rows in global memory for the float4 stores of d_tile
  const bool vec = K % 4 == 0 && aligned16(tile) && (!bwd || aligned16(d_tile));
  if (bwd) return vec ? fwfm_launch<true, true>(fn, tile, r, g, B, F, K, out, d_tile, d_r, st)
                      : fwfm_launch<true, false>(fn, tile, r, g, B, F, K, out, d_tile, d_r, st);
  return vec ? fwfm_launch<false, true>(fn, tile, r, g, B, F, K, out, d_tile, d_r, st)
             : fwfm_launch<false, false>(fn, tile, r, g, B, F, K, out, d_tile, d_r, st);
}

extern "C" int ctr_fwfm_fwd(const float* tile, const float* r, int64_t B, int64_t F, int64_t K, float* out, void* stream) {
  CTR_REQUIRE(tile && r && out, "ctr_fwfm_fwd: null argument");
  return fwfm_run(false, tile, r, nullptr, B, F, K, out, nullptr, nullptr, stream);
}

extern "C" int ctr_fwfm_bwd(const float* tile, const float* r, const float* g, int64_t B, int64_t F, int64_t K, float* d_tile,
                            float* d_r, void* stream) {
  CTR_REQUIRE(tile && r && g && d_tile && d_r, "ctr_fwfm_bwd: null argument");
  return fwfm_run(true, tile, r, g, B, F, K, nullptr, d_tile, d_r, stream);
}

extern "C" int ctr_afm_fwd(const float* tile, const float* w, const float* b, const float* h, int64_t B, int64_t F, int64_t K,
                           int64_t T, float* pooled, float* score, void* stream) {
  int rc = check_pw("ctr_afm_fwd", B, F, K);
  if (rc) return rc;
  CTR_REQUIRE(tile && w && b && h && pooled && T >= 1, "ctr_afm_fwd: null argument / bad attention_factor");
  CTR_REQUIRE(aligned16(tile), "ctr_afm_fwd: tile must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  return afm_dispatch<false>(tile, w, b, h, nullptr, B, F, K, T, pooled, score, nullptr, nullptr, nullptr, nullptr, as_stream(stream));
}

extern "C" int ctr_afm_bwd(const float* tile, const float* w, const float* b, const float* h, const float* g_pooled, int64_t B,
                           int64_t F, int64_t K, int64_t T, float* d_tile, float* d_w, float* d_b, float* d_h, void* stream) {
  int rc = check_pw("ctr_afm_bwd", B, F, K);
  if (rc) return rc;
  CTR_REQUIRE(tile && w && b && h && g_pooled && d_tile && d_w && d_b && d_h && T >= 1, "ctr_afm_bwd: null argument / bad attention_factor");
  CTR_REQUIRE(aligned16(tile), "ctr_afm_bwd: tile must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(d_w, 0, (size_t)K * T * sizeof(float), st));
  CTR_CUDA(cudaMemsetAsync(d_b, 0, (size_t)T * sizeof(float), st));
  CTR_CUDA(cudaMemsetAsync(d_h, 0, (size_t)T * sizeof(float), st));
  if (B == 0) return CTR_OK;
  return afm_dispatch<true>(tile, w, b, h, g_pooled, B, F, K, T, nullptr, nullptr, d_tile, d_w, d_b, d_h, st);
}

static int ffm_run(bool bwd, const float* tile, const float* g, int64_t B, int64_t F, int64_t K, float* out, float* d_tile, void* stream) {
  const char* fn = bwd ? "ctr_ffm_bwd" : "ctr_ffm_fwd";
  int rc = check_pw(fn, B, F, K);
  if (rc) return rc;
  CTR_REQUIRE(F * (F - 1) * K < (1LL << 30), "%s: F=%lld K=%lld too large", fn, (long long)F, (long long)K);
  if (B == 0) return CTR_OK;
  const int grid = capped_grid((B + 7) / 8, (long long)sm_count() * 8);
  if (bwd) return launch(fn, ffm_kernel<true>, grid, 256, 0, as_stream(stream), tile, g, (int)B, (int)F, (int)K, nullptr, d_tile);
  return launch(fn, ffm_kernel<false>, grid, 256, 0, as_stream(stream), tile, nullptr, (int)B, (int)F, (int)K, out, nullptr);
}

extern "C" int ctr_ffm_fwd(const float* tile, int64_t B, int64_t F, int64_t K, float* out, void* stream) {
  CTR_REQUIRE(tile && out, "ctr_ffm_fwd: null argument");
  return ffm_run(false, tile, nullptr, B, F, K, out, nullptr, stream);
}

extern "C" int ctr_ffm_bwd(const float* tile, const float* g, int64_t B, int64_t F, int64_t K, float* d_tile, void* stream) {
  CTR_REQUIRE(tile && g && d_tile, "ctr_ffm_bwd: null argument");
  return ffm_run(true, tile, g, B, F, K, nullptr, d_tile, stream);
}

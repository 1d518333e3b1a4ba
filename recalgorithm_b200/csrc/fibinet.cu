// Rows SENET and BILINEAR (SURVEY.md section 8a): FiBiNET's two interaction layers.
//
// Reference:
//   senet(input, embedding_dim, reduction_ratio)                   -- FiBiNET/senet.py:26-34
//       z = mean_K(x); a = relu(relu(z @ w1) @ w2); out = x * a[..., None]      (w1 (F,r), w2 (r,F), no bias)
//   bilinear_interaction_layer(input, embedding_dim, type, name)    -- FiBiNET/bilinear_interaction_layer.py:21-40
//       p_(i,j) = (x_i @ W) * x_j  for (i,j) in combinations(range(F-1), 2)  -> (B, (F-1)(F-2)/2, K)
//       W = w (K,K) ['all'] | w[i] ['each'] | w[pair index] ['interaction']
//
// H100 mapping: both layers are small, HBM/L2-bound CUDA-core kernels (K x K = 16 x 16 weights); SENET runs one
// warp per sample with the squeeze/excite vectors in shared memory, bilinear runs one CTA per sample with the
// sample's (F,K) block and the projected vectors in shared memory and writes the (P,K) output coalesced.
// Weight gradients are reduced per CTA in shared memory (or registers) and merged with fp32 atomics.
#include "ctr_common.cuh"

namespace ctr {

constexpr int SENET_WARPS = 4;

// smem layout per CTA: w1 (F*r) | w2 (r*F) | [bwd: dw1 (F*r) | dw2 (r*F)] | per warp: z (F), a1 (r), a2 (F), t1 (r), t2 (F)
template <bool BWD>
__global__ void __launch_bounds__(SENET_WARPS * 32)
senet_kernel(const float* __restrict__ x, const float* __restrict__ w1, const float* __restrict__ w2,
             const float* __restrict__ g, int B, int F, int K, int r, float* __restrict__ out /* fwd: out; bwd: dx */,
             float* __restrict__ dw1, float* __restrict__ dw2) {
  extern __shared__ __align__(16) float smem[];
  float* sw1 = smem;
  float* sw2 = sw1 + F * r;
  float* sdw1 = sw2 + r * F;
  float* sdw2 = BWD ? sdw1 + F * r : sdw1;
  float* per_warp = BWD ? sdw2 + r * F : sdw1;
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int stride = 3 * F + 2 * r;
  float* z = per_warp + wid * stride;
  float* a1 = z + F;
  float* a2 = a1 + r;
  float* t1 = a2 + F;      // bwd: da1
  float* t2 = t1 + r;      // bwd: da2, then dz
  for (int i = threadIdx.x; i < F * r; i += blockDim.x) {
    sw1[i] = __ldg(w1 + i); sw2[i] = __ldg(w2 + i);
    if (BWD) { sdw1[i] = 0.f; sdw2[i] = 0.f; }
  }
  __syncthreads();
  const float fK = (float)K;
  const int nwarps = gridDim.x * SENET_WARPS;
  for (int b = blockIdx.x * SENET_WARPS + wid; b < B; b += nwarps) {
    const float* xb = x + (size_t)b * F * K;
    const float* gb = BWD ? g + (size_t)b * F * K : nullptr;
    // squeeze: z[f] = mean_k x[f,k]   (+ bwd: t2[f] = sum_k g[f,k]*x[f,k])
    for (int f = lane; f < F; f += 32) {
      float s = 0.f, gx = 0.f;
      for (int k = 0; k < K; ++k) {
        const float v = __ldg(xb + f * K + k);
        s += v;
        if (BWD) gx += __ldg(gb + f * K + k) * v;
      }
      z[f] = s / fK;
      if (BWD) t2[f] = gx;
    }
    __syncwarp();
    for (int j = lane; j < r; j += 32) {
      float s = 0.f;
      for (int f = 0; f < F; ++f) s += z[f] * sw1[f * r + j];
      a1[j] = fmaxf(s, 0.f);
    }
    __syncwarp();
    for (int f = lane; f < F; f += 32) {
      float s = 0.f;
      for (int j = 0; j < r; ++j) s += a1[j] * sw2[j * F + f];
      a2[f] = fmaxf(s, 0.f);
    }
    __syncwarp();
    if (!BWD) {
      for (int i = lane; i < F * K; i += 32) out[(size_t)b * F * K + i] = __ldg(xb + i) * a2[i / K];
    } else {
      for (int f = lane; f < F; f += 32) t2[f] = a2[f] > 0.f ? t2[f] : 0.f;            // da2 (relu gate)
      __syncwarp();
      for (int j = lane; j < r; j += 32) {
        float s = 0.f;
        for (int f = 0; f < F; ++f) s += t2[f] * sw2[j * F + f];
        t1[j] = a1[j] > 0.f ? s : 0.f;                                                  // da1
      }
      __syncwarp();
      for (int i = lane; i < F * r; i += 32) {
        const int f1 = i / r, j1 = i % r;      // dw1[f,j] += z[f]*da1[j]
        atomicAdd(sdw1 + i, z[f1] * t1[j1]);
        const int j2 = i / F, f2 = i % F;      // dw2[j,f] += a1[j]*da2[f]
        atomicAdd(sdw2 + i, a1[j2] * t2[f2]);
      }
      __syncwarp();
      for (int f = lane; f < F; f += 32) {      // dz[f] = sum_j da1[j]*w1[f,j]  (overwrites t2 after its last use)
        float s = 0.f;
        for (int j = 0; j < r; ++j) s += t1[j] * sw1[f * r + j];
        z[f] = s / fK;                           // reuse z as dz/K
      }
      __syncwarp();
      for (int i = lane; i < F * K; i += 32)
        out[(size_t)b * F * K + i] = __ldg(gb + i) * a2[i / K] + z[i / K];
    }
    __syncwarp();
  }
  if (BWD) {
    __syncthreads();
    for (int i = threadIdx.x; i < F * r; i += blockDim.x) {
      atomicAdd(dw1 + i, sdw1[i]);
      atomicAdd(dw2 + i, sdw2[i]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// bilinear
// ---------------------------------------------------------------------------------------------------
constexpr int BIL_THREADS = 256;

__device__ __forceinline__ int pair_base(int i, int n) {   // index of pair (i, i+1) among combinations(range(n), 2)
  return i * (2 * n - i - 1) / 2;
}

// smem: xs (F*K) | vw ((F-1)*K)  [all/each]  | pair table (P x int2 packed as int)
template <int TYPE>
__global__ void __launch_bounds__(BIL_THREADS)
bilinear_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, int B, int F, int K,
                    float* __restrict__ out) {
  extern __shared__ __align__(16) float smem[];
  const int n = F - 1;                        // fields that take part (reference quirk: range(F-1))
  const int P = n * (n - 1) / 2;
  float* xs = smem;
  float* vw = xs + F * K;
  int* pairs = reinterpret_cast<int*>(vw + n * K);
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    for (int j = i + 1; j < n; ++j) pairs[pair_base(i, n) + (j - i - 1)] = (i << 16) | j;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    for (int i = threadIdx.x; i < F * K; i += blockDim.x) xs[i] = __ldg(x + (size_t)b * F * K + i);
    __syncthreads();
    if (TYPE != 2) {
      for (int t = threadIdx.x; t < n * K; t += blockDim.x) {
        const int i = t / K, k = t % K;
        const float* wi = TYPE == 0 ? w : w + (size_t)i * K * K;
        float s = 0.f;
        for (int c = 0; c < K; ++c) s += xs[i * K + c] * __ldg(wi + c * K + k);
        vw[t] = s;
      }
      __syncthreads();
      for (int t = threadIdx.x; t < P * K; t += blockDim.x) {
        const int p = t / K, k = t % K;
        const int ij = pairs[p];
        out[(size_t)b * P * K + t] = vw[(ij >> 16) * K + k] * xs[(ij & 0xffff) * K + k];
      }
    } else {
      for (int t = threadIdx.x; t < P * K; t += blockDim.x) {
        const int p = t / K, k = t % K;
        const int ij = pairs[p];
        const float* wp = w + (size_t)p * K * K;
        const float* xi = xs + (ij >> 16) * K;
        float s = 0.f;
        for (int c = 0; c < K; ++c) s += xi[c] * __ldg(wp + c * K + k);
        out[(size_t)b * P * K + t] = s * xs[(ij & 0xffff) * K + k];
      }
    }
  }
}

// Backward for 'all' / 'each'.  smem: xs (F*K) | vw (n*K) | dvw (n*K) | dwacc (TYPE0: K*K, TYPE1: n*K*K)
template <int TYPE>
__global__ void __launch_bounds__(BIL_THREADS)
bilinear_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ g, int B,
                    int F, int K, float* __restrict__ dx, float* __restrict__ dw) {
  extern __shared__ __align__(16) float smem[];
  const int n = F - 1;
  const int P = n * (n - 1) / 2;
  float* xs = smem;
  float* vw = xs + F * K;
  float* dvw = vw + n * K;
  float* dwacc = dvw + n * K;
  const int ndw = (TYPE == 0 ? 1 : n) * K * K;
  for (int i = threadIdx.x; i < ndw; i += blockDim.x) dwacc[i] = 0.f;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    for (int i = threadIdx.x; i < F * K; i += blockDim.x) xs[i] = __ldg(x + (size_t)b * F * K + i);
    __syncthreads();
    const float* gb = g + (size_t)b * P * K;
    for (int t = threadIdx.x; t < n * K; t += blockDim.x) {
      const int i = t / K, k = t % K;
      const float* wi = TYPE == 0 ? w : w + (size_t)i * K * K;
      float s = 0.f;
      for (int c = 0; c < K; ++c) s += xs[i * K + c] * __ldg(wi + c * K + k);
      vw[t] = s;
      // dvw_i[k] = sum_{j>i} g[(i,j),k] * x_j[k]
      float d = 0.f;
      const int p0 = pair_base(i, n);
      for (int j = i + 1; j < n; ++j) d += __ldg(gb + (size_t)(p0 + j - i - 1) * K + k) * xs[j * K + k];
      dvw[t] = d;
    }
    __syncthreads();
    // dx_j[k] = sum_{i<j} g[(i,j),k]*vw_i[k]  +  sum_c dvw_j[c] * W_j[k][c]   (second term only for j < n)
    for (int t = threadIdx.x; t < F * K; t += blockDim.x) {
      const int j = t / K, k = t % K;
      float s = 0.f;
      if (j < n) {
        for (int i = 0; i < j; ++i) s += __ldg(gb + (size_t)(pair_base(i, n) + j - i - 1) * K + k) * vw[i * K + k];
        const float* wj = TYPE == 0 ? w : w + (size_t)j * K * K;
        for (int c = 0; c < K; ++c) s += dvw[j * K + c] * __ldg(wj + k * K + c);
      }
      dx[(size_t)b * F * K + t] = s;           // field F-1 never takes part -> zero gradient
    }
    // dW_i[c][k] += x_i[c] * dvw_i[k]   (thread-owned accumulators: element e belongs to thread e % blockDim)
    for (int e = threadIdx.x; e < ndw; e += blockDim.x) {
      const int k = e % K, c = (e / K) % K;
      if (TYPE == 0) {
        float s = 0.f;
        for (int i = 0; i < n; ++i) s += xs[i * K + c] * dvw[i * K + k];
        dwacc[e] += s;
      } else {
        const int i = e / (K * K);
        dwacc[e] += xs[i * K + c] * dvw[i * K + k];
      }
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < ndw; e += blockDim.x) atomicAdd(dw + e, dwacc[e]);
}

// 'interaction' backward, data gradient: one CTA per sample.  smem: xs (F*K) | dxs (F*K) | dvw (P*K)
//   phase 1, thread (p,k): vw_p[k] = x_i . W_p[:,k];  dx_j[k] += g*vw;  dvw_p[k] = g*x_j[k]   (kept in smem)
//   phase 2, thread (p,c): dx_i[c] += dvw_p . W_p[c,:]
// (P*K shared atomics per phase instead of P*K*K in the first version.)
__global__ void __launch_bounds__(BIL_THREADS)
bilinear_bwd_interaction_dx_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                   const float* __restrict__ g, int B, int F, int K, float* __restrict__ dx) {
  extern __shared__ __align__(16) float smem[];
  const int n = F - 1;
  const int P = n * (n - 1) / 2;
  float* xs = smem;
  float* dxs = xs + F * K;
  float* dvw = dxs + F * K;
  int* pairs = reinterpret_cast<int*>(dvw + P * K);
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    for (int j = i + 1; j < n; ++j) pairs[pair_base(i, n) + (j - i - 1)] = (i << 16) | j;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    for (int i = threadIdx.x; i < F * K; i += blockDim.x) { xs[i] = __ldg(x + (size_t)b * F * K + i); dxs[i] = 0.f; }
    __syncthreads();
    const float* gb = g + (size_t)b * P * K;
    for (int t = threadIdx.x; t < P * K; t += blockDim.x) {
      const int p = t / K, k = t % K;
      const int ij = pairs[p];
      const int i = ij >> 16, j = ij & 0xffff;
      const float* wp = w + (size_t)p * K * K;
      float vwk = 0.f;
      for (int c = 0; c < K; ++c) vwk += xs[i * K + c] * __ldg(wp + c * K + k);
      const float gv = __ldg(gb + t);
      atomicAdd(dxs + j * K + k, gv * vwk);
      dvw[t] = gv * xs[j * K + k];
    }
    __syncthreads();
    for (int t = threadIdx.x; t < P * K; t += blockDim.x) {
      const int p = t / K, c = t % K;
      const float* wr = w + (size_t)p * K * K + (size_t)c * K;
      const float* dv = dvw + p * K;
      float sacc = 0.f;
      for (int k = 0; k < K; ++k) sacc += dv[k] * __ldg(wr + k);
      atomicAdd(dxs + (pairs[p] >> 16) * K + c, sacc);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < F * K; i += blockDim.x) dx[(size_t)b * F * K + i] = dxs[i];
  }
}

// 'interaction' backward, weight gradient: dW_p[c][k] = sum_b x[b,i,c] * g[b,p,k] * x[b,j,k].
// grid (P, nsplit); thread e = c*K + k loops over the samples of its split.
__global__ void __launch_bounds__(1024)
bilinear_bwd_interaction_dw_kernel(const float* __restrict__ x, const float* __restrict__ g, int B, int F, int K,
                                   float* __restrict__ dw) {
  const int n = F - 1;
  const int P = n * (n - 1) / 2;
  const int p = blockIdx.x;
  int i = 0;
  while (pair_base(i + 1, n) <= p && i + 1 < n - 1) ++i;
  const int j = i + 1 + (p - pair_base(i, n));
  for (int e = threadIdx.x; e < K * K; e += blockDim.x) {
    const int c = e / K, k = e % K;
    float s = 0.f;
    for (int b = blockIdx.y; b < B; b += gridDim.y) {
      const float* xb = x + (size_t)b * F * K;
      s += __ldg(xb + i * K + c) * __ldg(g + ((size_t)b * P + p) * K + k) * __ldg(xb + j * K + k);
    }
    atomicAdd(dw + (size_t)p * K * K + e, s);
  }
}


// ---------------------------------------------------------------------------------------------------
// bilinear, sample-batched "tournament" form (K = 8 / 16 / 32): the round-2 kernels.
//
// The first kernels above run one CTA per sample and fetch every pair's K x K weight from L2 for every sample (416 KB per
// sample for F = 30, K = 16, 'interaction'), and the 'interaction' weight gradient walks the batch with 4-byte strided loads:
// 1.86 ms for 122 MB of algorithmic traffic.  Here a CTA owns a TILE of samples (x staged in shared memory once) and a group
// of LP = K/KT lanes owns one pair at a time: a lane keeps KT columns and KT rows of the pair's weight in registers and reuses
// them for every sample of the tile.  The pairs are visited in the order of a round-robin tournament (circle method): the
// pairs of one round are field-disjoint, so inside a round every (sample, field, column) element of the shared dx tile has
// exactly ONE writer -- plain read-modify-writes, no shared-memory atomics; one block barrier per round.
//   fwd : vw[t] = x_i . W[:,k0+t] ; out[b,p,k0+t] = vw[t] * x_j[k0+t]
//   dx  : dx_j[k] += g*vw ; dv[k] = g*x_j[k] (exchanged inside the group through shared memory) ; dx_i[c] += dv . W[c,:]
//   dW  : second kernel, one CTA per (round, batch chunk): a lane accumulates KT rows of dW = sum_b x_i[c] * dv[:] in registers
//         over all samples of its chunk (no weights needed), one vector red per 4 elements at the end.
// KT (columns per lane) is the register-blocking knob: every x_i word a lane fetches from shared memory feeds KT FMAs, and the
// shared-memory -> register path (128 B/clk/SM, a broadcast LDS.128 still returns 512 B) is what bounds these kernels: with
// KT = 1 it is 4x oversubscribed against the FMA pipe (measured: fwd 60 us = the LDS time).
// The weight index of a pair is 0 ('all'), i ('each') or the pair index ('interaction').
// ---------------------------------------------------------------------------------------------------
struct RRShape {
  int n, np, rounds, slots, slot0;   // participating fields, padded to even, rounds = np-1, active slots per round, first slot
};

__host__ __device__ inline RRShape rr_shape(int F) {
  RRShape s;
  s.n = F - 1;
  s.np = (s.n & 1) ? s.n + 1 : s.n;
  s.rounds = s.np - 1;
  s.slot0 = (s.n & 1) ? 1 : 0;       // odd n: slot 0 would pair the round's field with the dummy -> skipped
  s.slots = s.np / 2 - s.slot0;
  return s;
}

// pair of (round r, slot) as (i << 16) | j with i < j
__device__ __forceinline__ int rr_pair(const RRShape& s, int r, int slot) {
  const int m1 = s.np - 1;
  const int sl = slot + s.slot0;
  int a, b;
  if (sl == 0) { a = r; b = s.np - 1; }
  else { a = (r + sl) % m1; b = (r - sl + m1) % m1; }
  return a < b ? (a << 16) | b : (b << 16) | a;
}

template <int K>
__device__ __forceinline__ void load_vec(float (&v)[K], const float* p) {      // p 16-byte aligned
#pragma unroll
  for (int q = 0; q < K / 4; ++q) {
    const float4 t = *reinterpret_cast<const float4*>(p + 4 * q);
    v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
  }
}

template <int KT, bool LDG = false>
__device__ __forceinline__ void ld_kt(float (&v)[KT], const float* p) {        // p aligned to KT floats
  if constexpr (KT == 1) {
    v[0] = LDG ? __ldg(p) : *p;
  } else if constexpr (KT == 2) {
    const float2 t = LDG ? __ldg(reinterpret_cast<const float2*>(p)) : *reinterpret_cast<const float2*>(p);
    v[0] = t.x; v[1] = t.y;
  } else {
    const float4 t = LDG ? __ldg(reinterpret_cast<const float4*>(p)) : *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  }
}

template <int KT>
__device__ __forceinline__ void st_kt(float* p, const float (&v)[KT]) {
  if constexpr (KT == 1) *p = v[0];
  else if constexpr (KT == 2) *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]);
  else *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}

template <int K>
__device__ __forceinline__ float dot_vec(const float (&a)[K], const float (&b)[K]) {
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int c = 0; c < K; c += 2) { s0 += a[c] * b[c]; s1 += a[c + 1] * b[c + 1]; }
  return s0 + s1;
}

__device__ __forceinline__ size_t rr_widx(int type, int i, int p) { return type == 0 ? 0 : type == 1 ? (size_t)i : (size_t)p; }

// smem: pair table (P ints, natural order) | xs (BS * F*K)
template <int K, int KT>
__global__ void __launch_bounds__(256)
bilinear_rr_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, int type, int B, int F, int BS,
                       float* __restrict__ out) {
  constexpr int LP = K / KT;
  extern __shared__ __align__(16) float smem[];
  const RRShape sh = rr_shape(F);
  const int n = sh.n, P = n * (n - 1) / 2, FK = F * K;
  // the forward has no accumulation conflicts: the groups of a warp take ADJACENT pairs, so a warp writes 32/LP * 4K contiguous
  // bytes of a sample's output row (the tournament order wrote 64-byte pieces 26 KB apart: 63 us = the DRAM rate of masked writes)
  int* tbl = reinterpret_cast<int*>(smem);
  float* xs = smem + ((P + 3) & ~3);
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    for (int j = i + 1; j < n; ++j) tbl[pair_base(i, n) + (j - i - 1)] = (i << 16) | j;
  const int grp = threadIdx.x / LP, k0 = (threadIdx.x % LP) * KT, G = blockDim.x / LP;
  const int ntiles = (B + BS - 1) / BS;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int b0 = tile * BS, bs = min(BS, B - b0);
    __syncthreads();
    for (int t = threadIdx.x; t < bs * FK / 4; t += blockDim.x)
      reinterpret_cast<float4*>(xs)[t] = __ldg(reinterpret_cast<const float4*>(x + (size_t)b0 * FK) + t);
    __syncthreads();
    // the weight columns of the group's NEXT pair are requested before the current pair is multiplied (first form: a third of the
    // stall samples sat on the first FMA after the weight loads)
    auto loadw = [&](int p, float (&wc)[KT][K]) {
      if (p < P) {
        const int ij = tbl[p];
        const float* wp = w + rr_widx(type, ij >> 16, p) * K * K;
#pragma unroll
        for (int c = 0; c < K; ++c) {
          float t[KT];
          ld_kt<KT, true>(t, wp + c * K + k0);
#pragma unroll
          for (int u = 0; u < KT; ++u) wc[u][c] = t[u];
        }
      }
    };
    auto run = [&](int p, const float (&wc)[KT][K]) {
      const int ij = tbl[p];
      const int i = ij >> 16, j = ij & 0xffff;
      float* ob = out + ((size_t)b0 * P + p) * K + k0;
#pragma unroll 2
      for (int s = 0; s < bs; ++s) {
        float xi[K], xj[KT], o[KT];
        load_vec<K>(xi, xs + s * FK + i * K);
        ld_kt<KT>(xj, xs + s * FK + j * K + k0);
#pragma unroll
        for (int u = 0; u < KT; ++u) o[u] = dot_vec<K>(xi, wc[u]) * xj[u];
        st_kt<KT>(ob + (size_t)s * P * K, o);
      }
    };
    float wa[KT][K], wb[KT][K];
    loadw(grp, wa);
    for (int p = grp; p < P; p += 2 * G) {
      loadw(p + G, wb);
      run(p, wa);
      if (p + G < P) {
        loadw(p + 2 * G, wa);
        run(p + G, wb);
      }
    }
  }
}

constexpr int RR_GP = 8;              // samples per tile of the dX kernel (their g values are prefetched into registers)

// smem: pair table | xs (BS*FK) | dxs (BS*FK) | dv exchange (groups * RR_GP * K).   BS <= RR_GP.
// A "step" is one (round, slot pass): every group holds one pair.  Each step runs two passes over the tile's samples:
//   pass A (needs the weight's columns + g):  dv = g*x_j -> exchange buffer ;  dx_j += g * (x_i . W[:,k])
//   pass B (needs the weight's rows):         dx_i += dv . W[c,:]
// so the global loads can be issued a pass ahead INTO THE SAME REGISTERS: the rows are requested before pass A, the NEXT step's
// columns and g values before pass B (first form: ncu attributed 17 % of the stall samples to the first use of g and ~18 % to the
// weight loads at the top of every step).
template <int K, int KT>
__global__ void __launch_bounds__(256)
bilinear_rr_bwd_dx_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ g, int type,
                          int B, int F, int BS, float* __restrict__ dx) {
  constexpr int LP = K / KT;
  extern __shared__ __align__(16) float smem[];
  const RRShape sh = rr_shape(F);
  const int n = sh.n, P = n * (n - 1) / 2, FK = F * K;
  int* tbl = reinterpret_cast<int*>(smem);
  float* xs = smem + ((sh.rounds * sh.slots + 3) & ~3);
  float* dxs = xs + (size_t)BS * FK;
  float* dvb = dxs + (size_t)BS * FK;
  for (int t = threadIdx.x; t < sh.rounds * sh.slots; t += blockDim.x) tbl[t] = rr_pair(sh, t / sh.slots, t % sh.slots);
  const int grp = threadIdx.x / LP, k0 = (threadIdx.x % LP) * KT, G = blockDim.x / LP;
  float* mydv = dvb + (size_t)grp * RR_GP * K;
  const int nslot_it = (sh.slots + G - 1) / G;          // same trip count for every group: the warp stays converged for __syncwarp
  const int NS = sh.rounds * nslot_it;
  auto pair_of = [&](int st, int& i, int& j, int& p, size_t& wi) -> bool {
    const int r = st / nslot_it, slot = grp + (st % nslot_it) * G;
    const bool act = slot < sh.slots;
    const int ij = act ? tbl[r * sh.slots + slot] : 1;
    i = ij >> 16; j = ij & 0xffff;
    p = pair_base(i, n) + (j - i - 1);
    wi = rr_widx(type, i, p);
    // idle groups load the weight / g of pair 0 but read the shared tiles at field F-1, which no pair ever writes (no stores at all)
    if (!act) i = j = F - 1;
    return act;
  };
  const int ntiles = (B + BS - 1) / BS;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int b0 = tile * BS, bs = min(BS, B - b0);
    __syncthreads();
    for (int t = threadIdx.x; t < bs * FK / 4; t += blockDim.x) {
      reinterpret_cast<float4*>(xs)[t] = __ldg(reinterpret_cast<const float4*>(x + (size_t)b0 * FK) + t);
      reinterpret_cast<float4*>(dxs)[t] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    float wcol[KT][K], wrow[KT][K], gq[RR_GP][KT];
    auto ld_cols_and_g = [&](int st) {
      int i, j, p;
      size_t wi;
      pair_of(st, i, j, p, wi);
      const float* wp = w + wi * K * K;
#pragma unroll
      for (int c = 0; c < K; ++c) {
        float t[KT];
        ld_kt<KT, true>(t, wp + c * K + k0);
#pragma unroll
        for (int u = 0; u < KT; ++u) wcol[u][c] = t[u];
      }
      const float* gb = g + ((size_t)b0 * P + p) * K + k0;
#pragma unroll
      for (int s = 0; s < RR_GP; ++s) {
        if (s < bs) ld_kt<KT, true>(gq[s], gb + (size_t)s * P * K);
        else {
#pragma unroll
          for (int t = 0; t < KT; ++t) gq[s][t] = 0.f;
        }
      }
    };
    ld_cols_and_g(0);
    for (int st = 0; st < NS; ++st) {
      int i, j, p;
      size_t wi;
      const bool act = pair_of(st, i, j, p, wi);
      {
        const float* wp = w + wi * K * K;
#pragma unroll
        for (int u = 0; u < KT; ++u) {
#pragma unroll
          for (int q = 0; q < K / 4; ++q) {
            const float4 t = __ldg(reinterpret_cast<const float4*>(wp + (k0 + u) * K) + q);
            wrow[u][4 * q] = t.x; wrow[u][4 * q + 1] = t.y; wrow[u][4 * q + 2] = t.z; wrow[u][4 * q + 3] = t.w;
          }
        }
      }
      __syncwarp();                                            // the previous step's pass B is done with the exchange buffer
#pragma unroll
      for (int s = 0; s < RR_GP; ++s) {                        // ---- pass A  (bs is uniform over the CTA)
        if (s < bs) {
          float xi[K], xj[KT], dvl[KT], dj[KT];
          load_vec<K>(xi, xs + s * FK + i * K);
          ld_kt<KT>(xj, xs + s * FK + j * K + k0);
          ld_kt<KT>(dj, dxs + s * FK + j * K + k0);
#pragma unroll
          for (int t = 0; t < KT; ++t) {
            dvl[t] = gq[s][t] * xj[t];
            dj[t] += gq[s][t] * dot_vec<K>(xi, wcol[t]);
          }
          st_kt<KT>(mydv + s * K + k0, dvl);
          if (act) st_kt<KT>(dxs + s * FK + j * K + k0, dj);
        }
      }
      __syncwarp();
      if (st + 1 < NS) ld_cols_and_g(st + 1);                  // into the registers pass A just finished with
#pragma unroll
      for (int s = 0; s < RR_GP; ++s) {                        // ---- pass B
        if (s < bs) {
          float dv[K], di[KT];
          load_vec<K>(dv, mydv + s * K);
          ld_kt<KT>(di, dxs + s * FK + i * K + k0);
#pragma unroll
          for (int t = 0; t < KT; ++t) di[t] += dot_vec<K>(dv, wrow[t]);
          if (act) st_kt<KT>(dxs + s * FK + i * K + k0, di);
        }
      }
      if ((st + 1) % nslot_it == 0) __syncthreads();           // next round: the same fields belong to other groups
    }
    for (int t = threadIdx.x; t < bs * FK / 4; t += blockDim.x)
      reinterpret_cast<float4*>(dx + (size_t)b0 * FK)[t] = reinterpret_cast<const float4*>(dxs)[t];
  }
}

// grid (pair blocks, chunks).  smem: dv exchange (groups * 2 * K).  x is read through L2 (7.9 MB at config size), g streams
// from HBM exactly once.
template <int K, int KT>
__global__ void __launch_bounds__(256)
bilinear_rr_bwd_dw_kernel(const float* __restrict__ x, const float* __restrict__ g, int type, int B, int F,
                          float* __restrict__ dw) {
  constexpr int LP = K / KT;
  constexpr int SUB = 8 / KT;                             // samples whose loads are issued together (even: the exchange buffers alternate)
  extern __shared__ __align__(16) float smem[];
  const int n = F - 1, P = n * (n - 1) / 2, FK = F * K;
  const int grp = threadIdx.x / LP, k0 = (threadIdx.x % LP) * KT, G = blockDim.x / LP;
  float* mydv = smem + grp * 2 * K;
  const int per = (B + gridDim.y - 1) / gridDim.y;
  const int b_lo = blockIdx.y * per, b_hi = min(B, b_lo + per);
  {
    // no accumulation conflicts here either: the groups of a CTA take ADJACENT pairs (a warp reads 32/LP * 4K contiguous bytes
    // of every sample's g row); idle groups of the last block shadow pair 0
    const int pp = blockIdx.x * G + grp;
    const bool act = pp < P;
    const int p = act ? pp : 0;
    int i = 0;
    while (i + 1 < n - 1 && pair_base(i + 1, n) <= p) ++i;
    const int j = i + 1 + (p - pair_base(i, n));
    float acc[KT][K];
#pragma unroll
    for (int t = 0; t < KT; ++t) {
#pragma unroll
      for (int k = 0; k < K; ++k) acc[t][k] = 0.f;
    }
    const float* xi_p = x + (size_t)i * K + k0;
    const float* xj_p = x + (size_t)j * K + k0;
    const float* g_p = g + (size_t)p * K + k0;
    // software pipeline: the loads of batch n+1 are issued before batch n is multiplied (first form: 81 % of the stall samples sat
    // on the first use of the loaded g / x_j values -- every batch waited a full DRAM latency)
    auto load = [&](int s0, float (&xi)[SUB][KT], float (&xj)[SUB][KT], float (&gv)[SUB][KT]) {
#pragma unroll
      for (int u = 0; u < SUB; ++u) {
        const int b = s0 + u;
        if (b < b_hi) {
          ld_kt<KT, true>(xi[u], xi_p + (size_t)b * FK);
          ld_kt<KT, true>(xj[u], xj_p + (size_t)b * FK);
          ld_kt<KT, true>(gv[u], g_p + (size_t)b * P * K);
        } else {
#pragma unroll
          for (int t = 0; t < KT; ++t) { xi[u][t] = 0.f; xj[u][t] = 0.f; gv[u][t] = 0.f; }
        }
      }
    };
    auto mult = [&](const float (&xi)[SUB][KT], const float (&xj)[SUB][KT], const float (&gv)[SUB][KT]) {
#pragma unroll
      for (int u = 0; u < SUB; ++u) {
        float dvl[KT];
#pragma unroll
        for (int t = 0; t < KT; ++t) dvl[t] = gv[u][t] * xj[u][t];
        float* buf = mydv + (u & 1) * K;
        st_kt<KT>(buf + k0, dvl);
        __syncwarp();
        float dv[K];
        load_vec<K>(dv, buf);
#pragma unroll
        for (int t = 0; t < KT; ++t) {
#pragma unroll
          for (int k = 0; k < K; ++k) acc[t][k] += xi[u][t] * dv[k];
        }
      }
    };
    float xa[SUB][KT], ja[SUB][KT], ga[SUB][KT], xb[SUB][KT], jb[SUB][KT], gb[SUB][KT];
    load(b_lo, xa, ja, ga);
    for (int s0 = b_lo; s0 < b_hi; s0 += 2 * SUB) {          // trip count is uniform over the CTA
      load(s0 + SUB, xb, jb, gb);
      mult(xa, ja, ga);
      load(s0 + 2 * SUB, xa, ja, ga);
      mult(xb, jb, gb);
    }
    if (act) {
      float* dst = dw + rr_widx(type, i, p) * K * K + (size_t)k0 * K;
#pragma unroll
      for (int t = 0; t < KT; ++t) {
#pragma unroll
        for (int q = 0; q < K / 4; ++q)
          atomicAdd(reinterpret_cast<float4*>(dst + t * K) + q,
                    make_float4(acc[t][4 * q], acc[t][4 * q + 1], acc[t][4 * q + 2], acc[t][4 * q + 3]));
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// bilinear 'all' / 'each', staged per-sample form (K = 8 / 16 / 32): the reference's default type is 'all'
// (FiBiNET/fibinet.py:45).  With one weight ('all') or one per field ('each') the projection vw_i = x_i W_i is computed once
// per field (n*K*K FMAs per sample instead of P*K*K) and the rest is element-wise over the (P,K) tile: these types want to be
// HBM streams.  The first kernels lost that to (1) runtime divisions `t / K, t % K` on every element, (2) 4-byte strided
// __ldg walks over g (twice per sample) and (3) un-overlapped loads.  Here K is a template parameter, the NEXT sample's x row
// and g tile are fetched with cp.async into a second buffer while the current one is processed, and both sweeps over g read
// the shared-memory copy.  One CTA works on one sample at a time; thread (f,k) owns dvw_f[k] and dx_f[k].
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void bl_cp_async16(float* smem_dst, const float* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void bl_cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bl_cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

constexpr int BST_THREADS = 512;

// smem: ws (nw*K*K) | xs[2] (F*K) | vw (n*K) | pair table (P ints)
template <int K, int TYPE>
__global__ void __launch_bounds__(BST_THREADS)
bilinear_st_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, int B, int F, float* __restrict__ out) {
  extern __shared__ __align__(16) float smem[];
  const int n = F - 1, P = n * (n - 1) / 2, FK = F * K;
  const int nw = TYPE == 0 ? 1 : n;
  float* ws = smem;
  float* xs = ws + nw * K * K;
  float* vw = xs + 2 * FK;
  int* pairs = reinterpret_cast<int*>(vw + n * K);
  for (int t = threadIdx.x; t < nw * K * K; t += blockDim.x) ws[t] = __ldg(w + t);
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    for (int j = i + 1; j < n; ++j) pairs[pair_base(i, n) + (j - i - 1)] = (i << 16) | j;
  int buf = 0;
  if (blockIdx.x < B)
    for (int t = threadIdx.x; t < FK / 4; t += blockDim.x) bl_cp_async16(xs + 4 * t, x + (size_t)blockIdx.x * FK + 4 * t);
  bl_cp_async_commit();
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    bl_cp_async_wait_all();
    __syncthreads();                                         // xs[buf] landed; vw of the previous sample is no longer read
    const int bn = b + gridDim.x;
    if (bn < B)
      for (int t = threadIdx.x; t < FK / 4; t += blockDim.x) bl_cp_async16(xs + (buf ^ 1) * FK + 4 * t, x + (size_t)bn * FK + 4 * t);
    bl_cp_async_commit();
    const float* xb = xs + buf * FK;
    for (int t = threadIdx.x; t < n * K; t += blockDim.x) {
      const int i = t / K, k = t % K;
      const float* wi = ws + (TYPE == 0 ? 0 : i * K * K);
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int c = 0; c < K; c += 2) { s0 += xb[i * K + c] * wi[c * K + k]; s1 += xb[i * K + c + 1] * wi[(c + 1) * K + k]; }
      vw[t] = s0 + s1;
    }
    __syncthreads();
    float4* ob = reinterpret_cast<float4*>(out + (size_t)b * P * K);
    for (int t = threadIdx.x; t < P * K / 4; t += blockDim.x) {
      const int p = t / (K / 4), k4 = (t % (K / 4)) * 4;
      const int ij = pairs[p];
      const float4 a = *reinterpret_cast<const float4*>(vw + (ij >> 16) * K + k4);
      const float4 c = *reinterpret_cast<const float4*>(xb + (ij & 0xffff) * K + k4);
      stg_stream_f4(ob + t, make_float4(a.x * c.x, a.y * c.y, a.z * c.z, a.w * c.w));
    }
    buf ^= 1;
  }
}

// smem: ws (nw*K*K) | dwacc (nw*K*K) | xs[2] (F*K) | gs[2] (P*K) | vw (n*K) | dvw (n*K)
template <int K, int TYPE>
__global__ void __launch_bounds__(BST_THREADS)
bilinear_st_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ g, int B, int F,
                       float* __restrict__ dx, float* __restrict__ dw) {
  extern __shared__ __align__(16) float smem[];
  const int n = F - 1, P = n * (n - 1) / 2, FK = F * K, PK = P * K;
  const int nw = TYPE == 0 ? 1 : n;
  float* ws = smem;
  float* dwacc = ws + nw * K * K;
  float* xs = dwacc + nw * K * K;
  float* gs = xs + 2 * FK;
  float* vw = gs + 2 * (size_t)PK;
  float* dvw = vw + n * K;
  for (int t = threadIdx.x; t < nw * K * K; t += blockDim.x) { ws[t] = __ldg(w + t); dwacc[t] = 0.f; }
  auto fetch = [&](int b, int bf) {
    for (int t = threadIdx.x; t < FK / 4; t += blockDim.x) bl_cp_async16(xs + bf * FK + 4 * t, x + (size_t)b * FK + 4 * t);
    for (int t = threadIdx.x; t < PK / 4; t += blockDim.x) bl_cp_async16(gs + (size_t)bf * PK + 4 * t, g + (size_t)b * PK + 4 * t);
  };
  int buf = 0;
  if (blockIdx.x < B) fetch(blockIdx.x, 0);
  bl_cp_async_commit();
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    bl_cp_async_wait_all();
    __syncthreads();                                         // this sample's tiles landed; vw / dvw of the previous one are free
    const int bn = b + gridDim.x;
    if (bn < B) fetch(bn, buf ^ 1);
    bl_cp_async_commit();
    const float* xb = xs + buf * FK;
    const float* gb = gs + (size_t)buf * PK;
    // sweep 1, thread (i,k): vw_i[k] = x_i . W_i[:,k] ;  dvw_i[k] = sum_{j>i} g[(i,j),k] * x_j[k]   (pairs of i are contiguous)
    for (int t = threadIdx.x; t < n * K; t += blockDim.x) {
      const int i = t / K, k = t % K;
      const float* wi = ws + (TYPE == 0 ? 0 : i * K * K);
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int c = 0; c < K; c += 2) { s0 += xb[i * K + c] * wi[c * K + k]; s1 += xb[i * K + c + 1] * wi[(c + 1) * K + k]; }
      vw[t] = s0 + s1;
      const float* gp = gb + pair_base(i, n) * K + k;
      float d0 = 0.f, d1 = 0.f;
      int j = i + 1;
      for (; j + 1 < n; j += 2) {
        d0 += gp[(j - i - 1) * K] * xb[j * K + k];
        d1 += gp[(j - i) * K] * xb[(j + 1) * K + k];
      }
      if (j < n) d0 += gp[(j - i - 1) * K] * xb[j * K + k];
      dvw[t] = d0 + d1;
    }
    __syncthreads();
    // sweep 2, thread (j,k): dx_j[k] = sum_{i<j} g[(i,j),k]*vw_i[k] + sum_c dvw_j[c] * W_j[k][c]   (field F-1: zero)
    for (int t = threadIdx.x; t < FK; t += blockDim.x) {
      const int j = t / K, k = t % K;
      float s0 = 0.f, s1 = 0.f;
      if (j < n) {
        // pair (i,j) sits at pair_base(i) + j - i - 1 and pair_base(i+1) - pair_base(i) = n - i - 1: walk the column with a
        // shrinking stride instead of re-deriving the index (the integer work was most of this loop's instructions)
        const float* gp = gb + (j - 1) * K + k;
        const float* vp = vw + k;
        int stride = (n - 2) * K;
        int i = 0;
        for (; i + 1 < j; i += 2) {
          s0 += gp[0] * vp[0];
          s1 += gp[stride] * vp[K];
          gp += 2 * stride - K;
          stride -= 2 * K;
          vp += 2 * K;
        }
        if (i < j) s0 += gp[0] * vp[0];
        const float* wj = ws + (TYPE == 0 ? 0 : j * K * K) + k * K;
#pragma unroll
        for (int c = 0; c < K; c += 2) { s0 += dvw[j * K + c] * wj[c]; s1 += dvw[j * K + c + 1] * wj[c + 1]; }
      }
      dx[(size_t)b * FK + t] = s0 + s1;
    }
    // dW_i[c][k] += x_i[c] * dvw_i[k]   (element e is always visited by the same thread: private accumulators in smem)
    for (int e = threadIdx.x; e < nw * K * K; e += blockDim.x) {
      const int k = e % K, c = (e / K) % K;
      if (TYPE == 0) {
        float s0 = 0.f, s1 = 0.f;
        int i = 0;
        for (; i + 1 < n; i += 2) { s0 += xb[i * K + c] * dvw[i * K + k]; s1 += xb[(i + 1) * K + c] * dvw[(i + 1) * K + k]; }
        if (i < n) s0 += xb[i * K + c] * dvw[i * K + k];
        dwacc[e] += s0 + s1;
      } else {
        const int i = e / (K * K);
        dwacc[e] += xb[i * K + c] * dvw[i * K + k];
      }
    }
    buf ^= 1;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < nw * K * K; e += blockDim.x) atomicAdd(dw + e, dwacc[e]);
}


static int g_bilinear_rr = 4;          // bit t: type t runs the tournament kernels (ctr_bilinear_set_rr); default: 'interaction' only
static int g_bilinear_old = 0;         // 1: 'all' / 'each' use the round-1 CTA-per-sample kernels instead of the staged ones
static int g_bilinear_tile = 0;        // tuning: samples per tile (0 = chosen from the shared-memory budget)
static int g_bilinear_kt = 0;          // tuning: weight columns per lane (0 = default for K)

static int rr_kt(int K) {
  int kt = g_bilinear_kt > 0 ? g_bilinear_kt : 2;
  while (kt > 1 && (K * kt > 64 || K / kt < 2)) kt >>= 1;      // <= 64 weight registers per operand, >= 2 lanes per pair
  return kt;
}

// threads of a tournament CTA: as many (K/kt)-lane groups as one round has pairs, at most 256 threads, whole warps
static int rr_threads(int F, int K, int kt) {
  const RRShape sh = rr_shape(F);
  const int lp = K / kt;
  int G = sh.slots < 256 / lp ? sh.slots : 256 / lp;
  if (G < 1) G = 1;
  return (G * lp + 31) / 32 * 32;
}

// samples per tile so that `arrays` staged copies of the tile fit `budget` bytes (0: not even one sample fits)
static int rr_tile(int F, int K, int arrays, size_t fixed, size_t budget) {
  int bs = g_bilinear_tile > 0 ? g_bilinear_tile : 8;
  while (bs >= 1 && fixed + (size_t)arrays * bs * F * K * sizeof(float) > budget) bs >>= 1;
  return bs;
}

// f(K, KT) for the tournament kernels of K in {8, 16, 32}: kt 1 and 2 as given, any other kt as 4 (K <= 16) or 2 (K = 32)
template <class Fn>
static int with_rr(int64_t K, int kt, Fn&& f) {
  return with_const<8, 16, 32>((int)K, [&](auto KK) {
    const int KT = kt == 1 || kt == 2 ? kt : KK <= 16 ? 4 : 2;
    if constexpr (KK <= 16) return with_const<1, 2, 4>(KT, [&](auto T) { return f(KK, T); });
    else return with_const<1, 2>(KT, [&](auto T) { return f(KK, T); });
  });
}

}  // namespace ctr

using namespace ctr;

static int check_senet(const char* fn, int64_t B, int64_t F, int64_t K, int64_t r) {
  CTR_REQUIRE(B >= 0 && F >= 1 && K >= 1 && r >= 1, "%s: bad sizes", fn);
  // reference: assert reduction_dim < embedding_dim (FiBiNET/senet.py:19)
  CTR_REQUIRE(r < K, "%s: reduction_dim must be less than embedding_dim (r=%lld, K=%lld)", fn, (long long)r, (long long)K);
  CTR_UNSUPPORTED(F > 1024 || K > 1024 || F * r > 8192, "%s: F=%lld K=%lld r=%lld too large", fn, (long long)F,
                  (long long)K, (long long)r);
  return CTR_OK;
}

extern "C" int ctr_senet_fwd(const float* x, const float* w1, const float* w2, int64_t B, int64_t F, int64_t K, int64_t r,
                             float* out, void* stream) {
  int rc = check_senet("ctr_senet_fwd", B, F, K, r);
  if (rc) return rc;
  CTR_REQUIRE(x && w1 && w2 && out, "ctr_senet_fwd: null argument");
  if (B == 0) return CTR_OK;
  const size_t smem = sizeof(float) * (2 * F * r + SENET_WARPS * (3 * F + 2 * r));
  return launch("ctr_senet_fwd", senet_kernel<false>, capped_grid((B + SENET_WARPS - 1) / SENET_WARPS, (long long)sm_count() * 8),
                SENET_WARPS * 32, smem, as_stream(stream), x, w1, w2, nullptr, (int)B, (int)F, (int)K, (int)r, out, nullptr, nullptr);
}

extern "C" int ctr_senet_bwd(const float* x, const float* w1, const float* w2, const float* g_out, int64_t B, int64_t F,
                             int64_t K, int64_t r, float* dx, float* dw1, float* dw2, void* stream) {
  int rc = check_senet("ctr_senet_bwd", B, F, K, r);
  if (rc) return rc;
  CTR_REQUIRE(x && w1 && w2 && g_out && dx && dw1 && dw2, "ctr_senet_bwd: null argument");
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(dw1, 0, sizeof(float) * F * r, st));
  CTR_CUDA(cudaMemsetAsync(dw2, 0, sizeof(float) * F * r, st));
  if (B == 0) return CTR_OK;
  const size_t smem = sizeof(float) * (4 * F * r + SENET_WARPS * (3 * F + 2 * r));
  return launch("ctr_senet_bwd", senet_kernel<true>, capped_grid((B + SENET_WARPS - 1) / SENET_WARPS, (long long)sm_count() * 4),
                SENET_WARPS * 32, smem, st, x, w1, w2, g_out, (int)B, (int)F, (int)K, (int)r, dx, dw1, dw2);
}


// the tournament kernels need K in {8,16,32} and 16-byte aligned arrays
static bool rr_usable(int64_t K, int type, const void* a, const void* b, const void* c, const void* d) {
  if (!((g_bilinear_rr >> type) & 1)) return false;
  if (K != 8 && K != 16 && K != 32) return false;
  return aligned16(a) && aligned16(b) && aligned16(c) && (d == nullptr || aligned16(d));
}

// the staged per-sample kernels ('all' / 'each'): K in {8,16,32}, 16-byte aligned arrays
static bool st_usable(int64_t K, int type, const void* a, const void* b, const void* c, const void* d) {
  if (g_bilinear_old || type > 1) return false;
  if (K != 8 && K != 16 && K != 32) return false;
  return aligned16(a) && aligned16(b) && aligned16(c) && (d == nullptr || aligned16(d));
}

extern "C" int ctr_bilinear_set_rr(int mask) {
  const int prev = g_bilinear_rr | (g_bilinear_old << 3) | (g_bilinear_tile << 4) | (g_bilinear_kt << 10);
  g_bilinear_rr = mask & 7;
  g_bilinear_old = (mask >> 3) & 1;
  g_bilinear_tile = (mask >> 4) & 63;                        // tuning only: samples per tile, 0 = automatic
  g_bilinear_kt = (mask >> 10) & 7;                          // tuning only: weight columns per lane (1, 2, 4), 0 = automatic
  return prev;
}

static int check_bilinear(const char* fn, int64_t B, int64_t F, int64_t K, int type) {
  CTR_REQUIRE(B >= 0 && F >= 1 && K >= 1, "%s: bad sizes", fn);
  // reference: ValueError for an unknown type (FiBiNET/bilinear_interaction_layer.py:36-38)
  CTR_REQUIRE(type >= 0 && type <= 2, "%s: Bilinear Interaction type must be in ['all','each','interaction'] (0..2), got %d",
              fn, type);
  CTR_UNSUPPORTED(F > 256 || K > 128, "%s: F=%lld K=%lld too large", fn, (long long)F, (long long)K);
  return CTR_OK;
}

extern "C" int ctr_bilinear_fwd(const float* x, const float* w, int64_t B, int64_t F, int64_t K, int type, float* out,
                                void* stream) {
  int rc = check_bilinear("ctr_bilinear_fwd", B, F, K, type);
  if (rc) return rc;
  CTR_REQUIRE(x && w && out, "ctr_bilinear_fwd: null argument");
  const int64_t n = F - 1, P = n * (n - 1) / 2;
  if (B == 0 || P == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  if (rr_usable(K, type, x, w, out, nullptr)) {
    const RRShape sh = rr_shape((int)F);
    const size_t fixed = sizeof(int) * ((sh.rounds * sh.slots + 3) & ~3);      // rounds * slots == P
    int bs = rr_tile((int)F, (int)K, 1, fixed, 64 * 1024);
    if (bs < 1) bs = rr_tile((int)F, (int)K, 1, fixed, 200 * 1024);
    if (bs >= 1) {
      const size_t smem_rr = fixed + sizeof(float) * bs * F * K;
      return with_rr(K, rr_kt((int)K), [&](auto KK, auto KT) {
        return launch_resident("ctr_bilinear_fwd", bilinear_rr_fwd_kernel<KK, KT>, (B + bs - 1) / bs, 256, smem_rr, st, x, w, type,
                               (int)B, (int)F, bs, out);
      });
    }
  }
  if (st_usable(K, type, x, w, out, nullptr)) {
    const int64_t nw = type == 0 ? 1 : n;
    const size_t smem_st = sizeof(float) * (nw * K * K + 2 * F * K + n * K) + sizeof(int) * P;
    if (smem_st <= 200 * 1024) {
      return with_const<8, 16, 32>((int)K, [&](auto KK) {
        return with_const<0, 1>(type, [&](auto T) {
          return launch_resident("ctr_bilinear_fwd", bilinear_st_fwd_kernel<KK, T>, B, BST_THREADS, smem_st, st, x, w, (int)B, (int)F,
                                 out);
        });
      });
    }
  }
  const size_t smem = sizeof(float) * (F * K + n * K) + sizeof(int) * P;
  return with_const<0, 1, 2>(type, [&](auto T) {
    return launch("ctr_bilinear_fwd", bilinear_fwd_kernel<T>, capped_grid(B, (long long)sm_count() * 8), BIL_THREADS, smem, st, x, w,
                  (int)B, (int)F, (int)K, out);
  });
}

extern "C" int ctr_bilinear_bwd(const float* x, const float* w, const float* g_out, int64_t B, int64_t F, int64_t K,
                                int type, float* dx, float* dw, void* stream) {
  int rc = check_bilinear("ctr_bilinear_bwd", B, F, K, type);
  if (rc) return rc;
  CTR_REQUIRE(x && w && g_out && dx && dw, "ctr_bilinear_bwd: null argument");
  const int64_t n = F - 1, P = n * (n - 1) / 2;
  const int64_t nw = (type == 0 ? 1 : type == 1 ? n : F * (F - 1) / 2) * K * K;
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * nw, st));
  if (B == 0) return CTR_OK;
  if (P == 0) {
    CTR_CUDA(cudaMemsetAsync(dx, 0, sizeof(float) * B * F * K, st));
    return CTR_OK;
  }
  if (rr_usable(K, type, x, w, dx, dw) && aligned16(g_out)) {
    const RRShape sh = rr_shape((int)F);
    const int kt = rr_kt((int)K);
    const int lp = (int)K / kt;
    const int threads = rr_threads((int)F, (int)K, kt);
    const size_t fixed = sizeof(int) * ((sh.rounds * sh.slots + 3) & ~3) + sizeof(float) * (threads / lp) * RR_GP * K;
    int bs = rr_tile((int)F, (int)K, 2, fixed, 72 * 1024);
    if (bs < 1) bs = rr_tile((int)F, (int)K, 2, fixed, 200 * 1024);
    if (bs > RR_GP) bs = RR_GP;                                  // the dX kernel keeps the tile's g values in registers
    if (bs >= 1) {
      const size_t smem_rr = fixed + sizeof(float) * 2 * bs * F * K;
      rc = with_rr(K, kt, [&](auto KK, auto KT) {
        return launch_resident("ctr_bilinear_bwd(dx)", bilinear_rr_bwd_dx_kernel<KK, KT>, (B + bs - 1) / bs, threads, smem_rr, st, x, w,
                               g_out, type, (int)B, (int)F, bs, dx);
      });
      if (rc) return rc;
      // weight gradient: one CTA per (block of adjacent pairs, batch chunk); ~8 CTAs per SM (the loads are latency-bound: ncu
      // long-scoreboard 12.6 per issue at 4), at least 32 samples per chunk
      const int dw_threads = 256, dw_groups = dw_threads / lp;
      const int pair_blocks = (int)((P + dw_groups - 1) / dw_groups);
      int chunks = (8 * sm_count() + pair_blocks - 1) / pair_blocks;
      const int max_chunks = (int)((B + 31) / 32);
      if (chunks > max_chunks) chunks = max_chunks;
      if (chunks < 1) chunks = 1;
      const size_t smem_dw = sizeof(float) * dw_groups * 2 * K;
      return with_rr(K, kt, [&](auto KK, auto KT) {
        return launch("ctr_bilinear_bwd(dw)", bilinear_rr_bwd_dw_kernel<KK, KT>, dim3((unsigned)pair_blocks, (unsigned)chunks), dw_threads,
                      smem_dw, st, x, g_out, type, (int)B, (int)F, dw);
      });
    }
  }
  if (type == 2) {
    const size_t smem = sizeof(float) * (2 * F * K + P * K) + sizeof(int) * P;
    CTR_UNSUPPORTED(smem > 200 * 1024, "ctr_bilinear_bwd: F=%lld K=%lld needs %zu B of shared memory", (long long)F,
                    (long long)K, smem);
    rc = launch("ctr_bilinear_bwd(dx)", bilinear_bwd_interaction_dx_kernel, capped_grid(B, (long long)sm_count() * 8), BIL_THREADS, smem, st,
                x, w, g_out, (int)B, (int)F, (int)K, dx);
    if (rc) return rc;
    int nsplit = (int)((B + 255) / 256);
    if (nsplit > 16) nsplit = 16;
    const int threads = (int)(K * K < 1024 ? ((K * K + 31) / 32) * 32 : 1024);
    return launch("ctr_bilinear_bwd(dw)", bilinear_bwd_interaction_dw_kernel, dim3((unsigned)P, (unsigned)nsplit), threads, 0, st, x, g_out,
                  (int)B, (int)F, (int)K, dw);
  }
  if (st_usable(K, type, x, w, dx, dw) && aligned16(g_out)) {
    const int64_t nw = type == 0 ? 1 : n;
    const size_t smem_st = sizeof(float) * (2 * nw * K * K + 2 * F * K + 2 * P * K + 2 * n * K);
    if (smem_st <= 200 * 1024) {
      return with_const<8, 16, 32>((int)K, [&](auto KK) {
        return with_const<0, 1>(type, [&](auto T) {
          return launch_resident("ctr_bilinear_bwd", bilinear_st_bwd_kernel<KK, T>, B, BST_THREADS, smem_st, st, x, w, g_out, (int)B,
                                 (int)F, dx, dw);
        });
      });
    }
  }
  const size_t smem = sizeof(float) * (F * K + 2 * n * K + (type == 0 ? 1 : n) * K * K);
  CTR_UNSUPPORTED(smem > 200 * 1024, "ctr_bilinear_bwd: F=%lld K=%lld needs %zu B of shared memory", (long long)F,
                  (long long)K, smem);
  return with_const<0, 1>(type, [&](auto T) {     // type 2 took the interaction path above
    return launch("ctr_bilinear_bwd", bilinear_bwd_kernel<T>, capped_grid(B, (long long)sm_count() * 2), BIL_THREADS, smem, st, x, w,
                  g_out, (int)B, (int)F, (int)K, dx, dw);
  });
}

// SURVEY.md 8f.4 -- BST transformer block (BST/transformer_layer.py:6-79), the sequence sibling of the DIN attention unit.
//
// One CTA (256 threads) per sample, every intermediate of the block in shared memory; the backward kernel recomputes the
// forward (nothing but the layer's inputs is read from HBM) and keeps the weight gradients of the whole CTA in shared
// memory (each element owned by one thread: no atomics until the final flush).  Shapes are tiny (T <= 64, d <= 32,
// heads <= 8: BST runs T = 51, d = 8, 3 heads), so this is a CUDA-core kernel; the tensor pipe has nothing to chew on.
//
// Reference quirks kept on purpose (see oracle/layers_np.py:bst_transformer_fwd):
//   * every head projects to d_model = d_k (not d_k / heads); values get no position embedding; the residual after the
//     attention uses the position-embedded queries;
//   * the length mask is added along the QUERY axis ((B,1,T,1) broadcast): in float32, x + (-2^32) is the same number for
//     every |x| < 256, so a masked query row attends uniformly -- done here with the same float32 add;
//   * tf.contrib.layers.layer_norm normalises over T and d together (begin_norm_axis = 1), eps = 1e-12;
//   * padded positions are ordinary keys (no key mask).
//
// params / d_params packing (floats): position_embedding (max_length, d) | w_q (H,d,d) | w_k | w_v | w_o (H*d, d) |
//   ln1_beta (d) | ln1_gamma (d) | dense_kernel (d,d) | dense_bias (d) | ln2_beta (d) | ln2_gamma (d)
#include "ctr_common.cuh"

namespace ctr {

constexpr int BST_NT = 256;

struct BstLayout {
  int pos, wq, wk, wv, wo, b1, g1, wd, bd, b2, g2, total;
};

__host__ __device__ inline BstLayout bst_layout(int d, int H, int maxlen) {
  BstLayout L;
  L.pos = 0;
  L.wq = maxlen * d;
  L.wk = L.wq + H * d * d;
  L.wv = L.wk + H * d * d;
  L.wo = L.wv + H * d * d;
  L.b1 = L.wo + H * d * d;
  L.g1 = L.b1 + d;
  L.wd = L.g1 + d;
  L.bd = L.wd + d * d;
  L.b2 = L.bd + d;
  L.g2 = L.b2 + d;
  L.total = L.g2 + d;
  return L;
}

// ---- tiny shared-memory GEMMs, all threads of the CTA.  Every matrix has D (= d_k = d_model) columns or D-long rows, so the
// helpers are specialised on D: one thread produces 4 adjacent outputs from one scalar + one 128-bit shared load per step
// (mm_nn / mm_tn), or one warp owns an output row with its D-long left operand in registers (mm_nt).  Leading dimensions
// are multiples of 4 floats; Q/K/V rows are padded to D + 4 so that eight consecutive rows start in eight different banks.
__device__ __forceinline__ void fma4(float4& s, float a, const float4& b) {
  s.x = fmaf(a, b.x, s.x); s.y = fmaf(a, b.y, s.y); s.z = fmaf(a, b.z, s.z); s.w = fmaf(a, b.w, s.w);
}
// C[t][0:D] (=|+=) sum_k A[t][k] * B[k][0:D]        (t < T, k < K)
template <int D>
__device__ __forceinline__ void mm_nn(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int T, int K, bool acc) {
  constexpr int D4 = D / 4;
  for (int e = threadIdx.x; e < T * D4; e += BST_NT) {
    const int t = e / D4, j = (e % D4) * 4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    const float* a = A + t * lda;
    const float* b = B + j;
    for (int k = 0; k < K; ++k) fma4(s, a[k], *reinterpret_cast<const float4*>(b + k * ldb));
    float4* c = reinterpret_cast<float4*>(C + t * ldc + j);
    if (acc) { const float4 o = *c; s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w; }
    *c = s;
  }
}
// C[k][0:D] (=|+=) sum_t A[t][k] * B[t][0:D]        (k < K, t < T)
template <int D>
__device__ __forceinline__ void mm_tn(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int T, int K, bool acc) {
  constexpr int D4 = D / 4;
  for (int e = threadIdx.x; e < K * D4; e += BST_NT) {
    const int k = e / D4, j = (e % D4) * 4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int t = 0; t < T; ++t) fma4(s, A[t * lda + k], *reinterpret_cast<const float4*>(B + t * ldb + j));
    float4* c = reinterpret_cast<float4*>(C + k * ldc + j);
    if (acc) { const float4 o = *c; s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w; }
    *c = s;
  }
}
// C[t][u] (=|+=) scale * sum_{k<D} A[t][k] * B[u][k]   (t < T, u < N): warp per row t, lanes over u
template <int D>
__device__ __forceinline__ void mm_nt(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int T, int N, float scale,
                                      bool acc) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = warp; t < T; t += BST_NT / 32) {
    float4 a[D / 4];
#pragma unroll
    for (int q = 0; q < D / 4; ++q) a[q] = *reinterpret_cast<const float4*>(A + t * lda + 4 * q);
    for (int u = lane; u < N; u += 32) {
      float s = 0.f;
#pragma unroll
      for (int q = 0; q < D / 4; ++q) {
        const float4 b = *reinterpret_cast<const float4*>(B + u * ldb + 4 * q);
        s = fmaf(a[q].x, b.x, s); s = fmaf(a[q].y, b.y, s); s = fmaf(a[q].z, b.z, s); s = fmaf(a[q].w, b.w, s);
      }
      C[t * ldc + u] = acc ? C[t * ldc + u] + scale * s : scale * s;
    }
  }
}

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();                                    // red[] may still be read from the previous reduction
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < BST_NT / 32; ++w) s += red[w];
  return s;
}

// layer norm over the whole (T, d) block: x -> xhat (in place), returns r = 1/sqrt(var + eps); y = xhat * gamma + beta
__device__ __forceinline__ float ln_forward(float* x, int n, float* red) {
  float s = 0.f;
  for (int e = threadIdx.x; e < n; e += BST_NT) s += x[e];
  const float mean = block_sum(s, red) / (float)n;
  float q = 0.f;
  for (int e = threadIdx.x; e < n; e += BST_NT) { const float c = x[e] - mean; q = fmaf(c, c, q); }
  const float var = block_sum(q, red) / (float)n;
  const float r = 1.f / sqrtf(var + 1e-12f);
  for (int e = threadIdx.x; e < n; e += BST_NT) x[e] = (x[e] - mean) * r;
  __syncthreads();
  return r;
}

// dxhat (in `g`, already multiplied by gamma) -> dx (in place): r * (dxhat - mean(dxhat) - xhat * mean(dxhat * xhat))
__device__ __forceinline__ void ln_backward(float* g, const float* xhat, float r, int n, float* red) {
  float a = 0.f, b = 0.f;
  for (int e = threadIdx.x; e < n; e += BST_NT) { a += g[e]; b = fmaf(g[e], xhat[e], b); }
  const float m1 = block_sum(a, red) / (float)n;
  const float m2 = block_sum(b, red) / (float)n;
  for (int e = threadIdx.x; e < n; e += BST_NT) g[e] = r * (g[e] - m1 - xhat[e] * m2);
  __syncthreads();
}

struct BstSmem {
  float *w, *gw, *xq, *xk, *xv, *Q, *K, *V, *A, *cat, *xh1, *f, *red;
  // backward only
  float *G, *dS, *dC, *dQ, *dK, *dV, *dxq, *dxk, *dxv;
};

__host__ __device__ inline int bst_tt(int T) { return (T * (T + 1) + 3) & ~3; }

__host__ __device__ inline size_t bst_smem_floats(int T, int d, int H, int total, bool bwd) {
  const int Td = T * d, Tp = T * (d + 4), TT = bst_tt(T);
  size_t n = (size_t)total + 3 * Td + 3 * Tp + TT + (size_t)T * H * d + 2 * Td + 32;
  if (bwd) n += (size_t)total + Td + TT + (size_t)T * H * d + 3 * Td + 3 * Td;
  return n;
}

__device__ inline BstSmem bst_carve(float* sm, int T, int d, int H, int total, bool bwd) {
  const int Td = T * d, Tp = T * (d + 4), TT = bst_tt(T);
  BstSmem s;
  float* p = sm;
  s.w = p; p += total;
  s.xq = p; p += Td; s.xk = p; p += Td; s.xv = p; p += Td;
  s.Q = p; p += Tp; s.K = p; p += Tp; s.V = p; p += Tp;
  s.A = p; p += TT;
  s.cat = p; p += T * H * d;
  s.xh1 = p; p += Td; s.f = p; p += Td;
  s.red = p; p += 32;
  if (bwd) {
    s.gw = p; p += total;
    s.G = p; p += Td;
    s.dS = p; p += TT;
    s.dC = p; p += T * H * d;
    s.dQ = p; p += Td; s.dK = p; p += Td; s.dV = p; p += Td;
    s.dxq = p; p += Td; s.dxk = p; p += Td; s.dxv = p; p += Td;
  } else {
    s.gw = s.G = s.dS = s.dC = s.dQ = s.dK = s.dV = s.dxq = s.dxk = s.dxv = nullptr;
  }
  return s;
}

// Q, K, V of head h and A = softmax(Q K^T / sqrt(d) + query-axis mask)
template <int D>
__device__ __forceinline__ void bst_head_forward(const BstSmem& s, const BstLayout& L, int h, int T, int len) {
  constexpr int dp = D + 4;
  const int tp = T + 1;
  mm_nn<D>(s.xq, D, s.w + L.wq + h * D * D, D, s.Q, dp, T, D, false);
  mm_nn<D>(s.xk, D, s.w + L.wk + h * D * D, D, s.K, dp, T, D, false);
  mm_nn<D>(s.xv, D, s.w + L.wv + h * D * D, D, s.V, dp, T, D, false);
  __syncthreads();
  mm_nt<D>(s.Q, dp, s.K, dp, s.A, tp, T, T, 1.f / sqrtf((float)D), false);      // tf.matmul(Q, K_T) / math.sqrt(d_k)
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int t = warp; t < T; t += BST_NT / 32) {
    float* row = s.A + t * tp;
    const bool masked = t >= len;
    float mx = -INFINITY;
    for (int u = lane; u < T; u += 32) {
      float v = row[u];
      if (masked) { v = __fadd_rn(v, -4294967296.f); row[u] = v; }             // float32(-2**32 + 1): collapses the row (see header)
      mx = fmaxf(mx, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float den = 0.f;
    for (int u = lane; u < T; u += 32) { const float ex = expf(row[u] - mx); row[u] = ex; den += ex; }
    den = warp_sum(den);
    const float inv = 1.f / den;
    for (int u = lane; u < T; u += 32) row[u] *= inv;
  }
  __syncthreads();
}

template <int D, bool BWD>
__global__ void __launch_bounds__(BST_NT, D <= 16 ? (BWD ? 3 : 4) : 1)
bst_kernel(const float* __restrict__ queries, const float* __restrict__ keys, const float* __restrict__ values,
           const long long* __restrict__ keys_length, const float* __restrict__ params, const float* __restrict__ g_out, int B,
           int T, int H, int maxlen, int use_pos, float* __restrict__ out, float* __restrict__ d_queries,
           float* __restrict__ d_keys, float* __restrict__ d_values, float* __restrict__ d_params) {
  extern __shared__ __align__(16) float sm[];
  constexpr int d = D, dp = D + 4;
  const BstLayout L = bst_layout(d, H, maxlen);
  const BstSmem s = bst_carve(sm, T, d, H, L.total, BWD);
  const int Td = T * d, Hd = H * d, tp = T + 1;
  for (int e = threadIdx.x; e < L.total; e += BST_NT) { s.w[e] = __ldg(params + e); if (BWD) s.gw[e] = 0.f; }
  __syncthreads();
  const float f1 = 0.5f * (1.f + 0.01f), f2 = 0.5f * (1.f - 0.01f);      // BST/leakyrelu.py:14-16

  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    long long len64 = __ldg(keys_length + b);
    const int len = len64 < 0 ? 0 : (len64 > T ? T : (int)len64);
    for (int e = threadIdx.x; e < Td; e += BST_NT) {
      const float pe = use_pos ? s.w[L.pos + e] : 0.f;
      s.xq[e] = __ldg(queries + (size_t)b * Td + e) + pe;
      s.xk[e] = __ldg(keys + (size_t)b * Td + e) + pe;
      s.xv[e] = __ldg(values + (size_t)b * Td + e);
    }
    __syncthreads();
    // ---- attention, head by head -> cat (T, H*d)
    for (int h = 0; h < H; ++h) {
      bst_head_forward<D>(s, L, h, T, len);
      mm_nn<D>(s.A, tp, s.V, dp, s.cat + h * d, Hd, T, T, false);
      __syncthreads();
    }
    // ---- all_heads = cat @ w_o ; net = layer_norm(all_heads + queries)
    mm_nn<D>(s.cat, Hd, s.w + L.wo, d, s.xh1, d, T, Hd, false);
    __syncthreads();
    for (int e = threadIdx.x; e < Td; e += BST_NT) s.xh1[e] += s.xq[e];
    __syncthreads();
    const float r1 = ln_forward(s.xh1, Td, s.red);                         // xh1 = xhat1
    float* y1 = BWD ? s.dV : s.xk;                                         // scratch: xk is dead in the forward-only kernel
    for (int e = threadIdx.x; e < Td; e += BST_NT) y1[e] = fmaf(s.xh1[e], s.w[L.g1 + e % d], s.w[L.b1 + e % d]);
    __syncthreads();
    // ---- ffn = leakyrelu(dense(net)) ; out = layer_norm(ffn + net)
    mm_nn<D>(y1, d, s.w + L.wd, d, s.f, d, T, d, false);
    __syncthreads();
    float* n2 = BWD ? s.G : s.xq;                                          // xq is dead in the forward-only kernel
    for (int e = threadIdx.x; e < Td; e += BST_NT) {
      const float fv = s.f[e] + s.w[L.bd + e % d];
      s.f[e] = fv;
      n2[e] = f1 * fv + f2 * fabsf(fv) + y1[e];
    }
    __syncthreads();
    const float r2 = ln_forward(n2, Td, s.red);                            // n2 = xhat2
    if (!BWD) {
      for (int e = threadIdx.x; e < Td; e += BST_NT) out[(size_t)b * Td + e] = fmaf(n2[e], s.w[L.g2 + e % d], s.w[L.b2 + e % d]);
      __syncthreads();
      continue;
    }

    // =============================================================== backward ===============================================
    // ---- layer norm 2: G holds xhat2; load g, accumulate d_gamma2 / d_beta2, turn dn into d(n2)
    float* dn = s.dQ;                                                      // scratch (T,d): free until the head loop
    for (int e = threadIdx.x; e < Td; e += BST_NT) dn[e] = __ldg(g_out + (size_t)b * Td + e);
    __syncthreads();
    for (int j = threadIdx.x; j < d; j += BST_NT) {
      float a = 0.f, c = 0.f;
      for (int t = 0; t < T; ++t) { a = fmaf(dn[t * d + j], s.G[t * d + j], a); c += dn[t * d + j]; }
      s.gw[L.g2 + j] += a; s.gw[L.b2 + j] += c;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < Td; e += BST_NT) dn[e] *= s.w[L.g2 + e % d];
    __syncthreads();
    ln_backward(dn, s.G, r2, Td, s.red);                                   // dn = d(n2): gradient of ffn_out and (residual) of y1
    // ---- leaky relu + dense: df -> G ; d_dense_kernel, d_dense_bias ; dy1 = dn + df @ Wd^T -> dK scratch
    for (int e = threadIdx.x; e < Td; e += BST_NT) {
      const float fv = s.f[e];
      s.G[e] = dn[e] * (f1 + f2 * (fv > 0.f ? 1.f : (fv < 0.f ? -1.f : 0.f)));
    }
    __syncthreads();
    mm_tn<D>(y1, d, s.G, d, s.gw + L.wd, d, T, d, true);                   // d_kernel += y1^T df
    for (int j = threadIdx.x; j < d; j += BST_NT) {
      float a = 0.f;
      for (int t = 0; t < T; ++t) a += s.G[t * d + j];
      s.gw[L.bd + j] += a;
    }
    float* dy1 = s.dK;
    mm_nt<D>(s.G, d, s.w + L.wd, d, dy1, d, T, d, 1.f, false);            // df @ Wd^T
    __syncthreads();
    for (int e = threadIdx.x; e < Td; e += BST_NT) dy1[e] += dn[e];
    __syncthreads();
    // ---- layer norm 1
    for (int j = threadIdx.x; j < d; j += BST_NT) {
      float a = 0.f, c = 0.f;
      for (int t = 0; t < T; ++t) { a = fmaf(dy1[t * d + j], s.xh1[t * d + j], a); c += dy1[t * d + j]; }
      s.gw[L.g1 + j] += a; s.gw[L.b1 + j] += c;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < Td; e += BST_NT) dy1[e] *= s.w[L.g1 + e % d];
    __syncthreads();
    ln_backward(dy1, s.xh1, r1, Td, s.red);                                // dy1 = d(all_heads + queries)
    for (int e = threadIdx.x; e < Td; e += BST_NT) { s.G[e] = dy1[e]; s.dxq[e] = dy1[e]; s.dxk[e] = 0.f; s.dxv[e] = 0.f; }
    __syncthreads();
    // ---- w_o: d_w_o += cat^T @ G ; dC = G @ w_o^T
    mm_tn<D>(s.cat, Hd, s.G, d, s.gw + L.wo, d, T, Hd, true);
    mm_nt<D>(s.G, d, s.w + L.wo, d, s.dC, Hd, T, Hd, 1.f, false);
    __syncthreads();
    // ---- heads
    const float scale = 1.f / sqrtf((float)d);
    for (int h = 0; h < H; ++h) {
      bst_head_forward<D>(s, L, h, T, len);
      const float* dO = s.dC + h * d;                                      // (T, d) with leading dimension H*d
      mm_nt<D>(dO, Hd, s.V, dp, s.dS, tp, T, T, 1.f, false);              // dA[t][u] = sum_j dO[t][j] V[u][j]
      mm_tn<D>(s.A, tp, dO, Hd, s.dV, d, T, T, false);                     // dV[u][j] = sum_t A[t][u] dO[t][j]
      __syncthreads();
      {                                                                    // dS = A * (dA - rowsum(A * dA)) / sqrt(d)
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (int t = warp; t < T; t += BST_NT / 32) {
          float dot = 0.f;
          for (int u = lane; u < T; u += 32) dot = fmaf(s.A[t * tp + u], s.dS[t * tp + u], dot);
          dot = warp_sum(dot);
          for (int u = lane; u < T; u += 32) s.dS[t * tp + u] = s.A[t * tp + u] * (s.dS[t * tp + u] - dot) * scale;
        }
      }
      __syncthreads();
      mm_nn<D>(s.dS, tp, s.K, dp, s.dQ, d, T, T, false);                   // dQ = dS @ K
      mm_tn<D>(s.dS, tp, s.Q, dp, s.dK, d, T, T, false);                   // dK = dS^T @ Q
      __syncthreads();
      mm_tn<D>(s.xq, d, s.dQ, d, s.gw + L.wq + h * d * d, d, T, d, true);
      mm_tn<D>(s.xk, d, s.dK, d, s.gw + L.wk + h * d * d, d, T, d, true);
      mm_tn<D>(s.xv, d, s.dV, d, s.gw + L.wv + h * d * d, d, T, d, true);
      mm_nt<D>(s.dQ, d, s.w + L.wq + h * d * d, d, s.dxq, d, T, d, 1.f, true);
      mm_nt<D>(s.dK, d, s.w + L.wk + h * d * d, d, s.dxk, d, T, d, 1.f, true);
      mm_nt<D>(s.dV, d, s.w + L.wv + h * d * d, d, s.dxv, d, T, d, 1.f, true);
      __syncthreads();
    }
    for (int e = threadIdx.x; e < Td; e += BST_NT) {
      d_queries[(size_t)b * Td + e] = s.dxq[e];
      d_keys[(size_t)b * Td + e] = s.dxk[e];
      d_values[(size_t)b * Td + e] = s.dxv[e];
      if (use_pos) s.gw[L.pos + e] += s.dxq[e] + s.dxk[e];
    }
    __syncthreads();
  }
  if (BWD) {
    __syncthreads();
    for (int e = threadIdx.x; e < L.total; e += BST_NT)
      if (s.gw[e] != 0.f) atomicAdd(d_params + e, s.gw[e]);
  }
}

}  // namespace ctr

using namespace ctr;

static int bst_check(const char* fn, int64_t B, int64_t T, int64_t d, int64_t heads, int64_t max_length, int use_pos) {
  CTR_REQUIRE(B >= 0 && T >= 1 && d >= 1 && heads >= 1, "%s: bad sizes B=%lld T=%lld d=%lld heads=%lld", fn, (long long)B,
              (long long)T, (long long)d, (long long)heads);
  CTR_REQUIRE(max_length >= 1 && (!use_pos || max_length >= T), "%s: max_length=%lld must cover T=%lld (position embedding rows)",
              fn, (long long)max_length, (long long)T);
  CTR_UNSUPPORTED(T > 128 || d > 64 || heads > 16 || max_length > 4096, "%s: T=%lld d=%lld heads=%lld max_length=%lld beyond the "
                  "single-CTA kernel (T <= 128, d <= 64, heads <= 16)", fn, (long long)T, (long long)d, (long long)heads,
                  (long long)max_length);
  return CTR_OK;
}

extern "C" int64_t ctr_bst_param_count(int64_t d, int64_t heads, int64_t max_length) {
  if (d < 1 || heads < 1 || max_length < 1 || d > 4096 || heads > 4096 || max_length > (1 << 24)) return -1;
  return (int64_t)max_length * d + 4 * heads * d * d + d * d + 5 * d;
}

template <int D, bool BWD>
static int bst_launch_d(const char* fn, const float* q, const float* k, const float* v, const int64_t* len, const float* params,
                        const float* g, int64_t B, int64_t T, int64_t H, int64_t maxlen, int use_pos, float* out, float* dq,
                        float* dk, float* dv, float* dparams, cudaStream_t st) {
  const BstLayout L = bst_layout(D, (int)H, (int)maxlen);
  const size_t smem = bst_smem_floats((int)T, D, (int)H, L.total, BWD) * sizeof(float);
  CTR_UNSUPPORTED(smem > 220 * 1024, "%s: T=%lld d=%d heads=%lld max_length=%lld needs %zu bytes of shared memory per sample (limit 220 KB)",
                  fn, (long long)T, D, (long long)H, (long long)maxlen, smem);
  return launch_resident(fn, bst_kernel<D, BWD>, B, BST_NT, smem, st, q, k, v, reinterpret_cast<const long long*>(len), params, g,
                         (int)B, (int)T, (int)H, (int)maxlen, use_pos, out, dq, dk, dv, dparams);
}

template <bool BWD>
static int bst_launch(const char* fn, const float* q, const float* k, const float* v, const int64_t* len, const float* params,
                      const float* g, int64_t B, int64_t T, int64_t d, int64_t H, int64_t maxlen, int use_pos, float* out,
                      float* dq, float* dk, float* dv, float* dparams, cudaStream_t st) {
  CTR_UNSUPPORTED(d != 4 && d != 8 && d != 16 && d != 32 && d != 64, "%s: d=%lld unsupported (d_k in {4, 8, 16, 32, 64})", fn,
                  (long long)d);
  return with_const<4, 8, 16, 32, 64>((int)d, [&](auto D) {
    return bst_launch_d<D, BWD>(fn, q, k, v, len, params, g, B, T, H, maxlen, use_pos, out, dq, dk, dv, dparams, st);
  });
}

extern "C" int ctr_bst_transformer_fwd(const float* queries, const float* keys, const float* values, const int64_t* keys_length,
                                       const float* params, int64_t B, int64_t T, int64_t d, int64_t heads, int64_t max_length,
                                       int use_position_embedding, float* out, void* stream) {
  int rc = bst_check("ctr_bst_transformer_fwd", B, T, d, heads, max_length, use_position_embedding);
  if (rc) return rc;
  CTR_REQUIRE(queries && keys && values && keys_length && params && out, "ctr_bst_transformer_fwd: null argument");
  if (B == 0) return CTR_OK;
  return bst_launch<false>("ctr_bst_transformer_fwd", queries, keys, values, keys_length, params, nullptr, B, T, d, heads, max_length,
                           use_position_embedding, out, nullptr, nullptr, nullptr, nullptr, as_stream(stream));
}

extern "C" int ctr_bst_transformer_bwd(const float* queries, const float* keys, const float* values, const int64_t* keys_length,
                                       const float* params, const float* g_out, int64_t B, int64_t T, int64_t d, int64_t heads,
                                       int64_t max_length, int use_position_embedding, float* d_queries, float* d_keys,
                                       float* d_values, float* d_params, void* stream) {
  int rc = bst_check("ctr_bst_transformer_bwd", B, T, d, heads, max_length, use_position_embedding);
  if (rc) return rc;
  CTR_REQUIRE(queries && keys && values && keys_length && params && g_out && d_queries && d_keys && d_values && d_params,
              "ctr_bst_transformer_bwd: null argument");
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(d_params, 0, (size_t)ctr_bst_param_count(d, heads, max_length) * sizeof(float), st));
  if (B == 0) return CTR_OK;
  return bst_launch<true>("ctr_bst_transformer_bwd", queries, keys, values, keys_length, params, g_out, B, T, d, heads, max_length,
                          use_position_embedding, nullptr, d_queries, d_keys, d_values, d_params, st);
}

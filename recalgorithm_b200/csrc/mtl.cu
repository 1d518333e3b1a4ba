// Row MTL: multi-task loss balancing for MMoE / PLE -- the per-task sigmoid cross-entropies with the sum, GradNorm-weight
// and uncertainty-weight totals, the Gram matrix of the per-task gradients over the shared parameters, the PCGrad
// combination and the GradNorm weight update.  The definitions are in include/ctr_b200.h ("Row MTL") and DESIGN §2.
//
// Every reduction here has a fixed partition and a fixed summation order, so the same inputs give the same bits on every
// call: GradNorm divides these losses and norms by each other, and PCGrad branches on the sign of their dot products.
#include <cooperative_groups.h>

#include "ctr_common.cuh"

namespace cg = cooperative_groups;

namespace ctr {
namespace mtl {

constexpr int MAX_T = 8;
constexpr int CE_CTAS = 8;            // one cluster; every CTA takes 1/8 of every task's batch
constexpr int CE_THREADS = 512;
constexpr int GRAM_THREADS = 256;
constexpr int GRAM_COLS_PER_CTA = 2048;
constexpr int GRAM_MAX_CTAS = 1024;
constexpr int COMBINE_THREADS = 256;

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Per-task mean sigmoid cross-entropy (TF's stable form, as ctr_sigmoid_ce) and the method's total.  CTA r of the cluster
// sums elements [r*chunk, (r+1)*chunk) of every task in float64; CTA 0 adds the eight partials of each task in rank order
// through distributed shared memory.
__global__ void __cluster_dims__(CE_CTAS, 1, 1) __launch_bounds__(CE_THREADS)
multitask_ce_kernel(const float* __restrict__ logits, const float* __restrict__ labels, int T, int B, int method,
                    const float* __restrict__ task_param, float* __restrict__ task_loss, float* __restrict__ total,
                    float* __restrict__ d_logits, float* __restrict__ d_param) {
  __shared__ double s_warp[MAX_T][CE_THREADS / 32];
  __shared__ double s_part[MAX_T];
  __shared__ double s_term[MAX_T];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float inv_b = B > 0 ? 1.f / (float)B : 0.f;
  const int chunk = (int)(((int64_t)B + CE_CTAS - 1) / CE_CTAS);
  const int lo = (int)min((int64_t)rank * chunk, (int64_t)B), hi = (int)min((int64_t)lo + chunk, (int64_t)B);
  for (int t = 0; t < T; ++t) {
    const float* x_t = logits + (int64_t)t * B;
    const float* z_t = labels + (int64_t)t * B;
    float* d_t = d_logits != nullptr ? d_logits + (int64_t)t * B : nullptr;
    double acc = 0.0;
#pragma unroll 4
    for (int64_t i = lo + (int)threadIdx.x; i < hi; i += CE_THREADS) {
      const float x = __ldg(x_t + i), z = __ldg(z_t + i);
      acc += (double)(fmaxf(x, 0.f) - x * z + log1pf(expf(-fabsf(x))));
      if (d_t != nullptr) d_t[i] = (1.f / (1.f + expf(-x)) - z) * inv_b;
    }
    acc = warp_sum_d(acc);
    if (lane == 0) s_warp[t][warp] = acc;
  }
  __syncthreads();
  if (warp < T) {
    double v = lane < CE_THREADS / 32 ? s_warp[warp][lane] : 0.0;
    v = warp_sum_d(v);
    if (lane == 0) s_part[warp] = v;
  }
  cluster.sync();
  if (rank == 0) {
    if (threadIdx.x < T) {
      const int t = threadIdx.x;
      double sum = 0.0;
      for (int r = 0; r < CE_CTAS; ++r) sum += cluster.map_shared_rank(s_part, r)[t];
      const double L = B > 0 ? sum / (double)B : 0.0;
      double term = L, d = 0.0;
      if (method == 1) {
        term = (double)task_param[t] * L;
        d = L;
      } else if (method == 2) {
        const double s = (double)task_param[t], e = exp(-s);
        term = e * L + 0.5 * s;
        d = -e * L + 0.5;
      }
      task_loss[t] = (float)L;
      if (d_param != nullptr) d_param[t] = (float)d;
      s_term[t] = term;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double sum = 0.0;
      for (int t = 0; t < T; ++t) sum += s_term[t];
      total[0] = (float)sum;
    }
  }
  cluster.sync();  // the other CTAs' s_part stays alive until CTA 0 has read it
}

// The T(T+1)/2 pair index of i <= j, row-major over the upper triangle.
__host__ __device__ constexpr int num_pairs(int T) { return T * (T + 1) / 2; }

// Stage 1 of the Gram matrix: CTA g sums g_i[c] * g_j[c] over its columns c = (g + k*G)*256 + tid for every pair i <= j
// in float64 (the products of two floats are exact there) and writes its NP partials to partial[g][NP].
template <int T>
__global__ void __launch_bounds__(GRAM_THREADS)
gram_partial_kernel(const float* __restrict__ g, int64_t ld, int64_t P, double* __restrict__ partial) {
  constexpr int NP = num_pairs(T);
  __shared__ double s[GRAM_THREADS / 32][NP];
  double acc[NP];
#pragma unroll
  for (int p = 0; p < NP; ++p) acc[p] = 0.0;
  for (int64_t c = (int64_t)blockIdx.x * GRAM_THREADS + threadIdx.x; c < P; c += (int64_t)gridDim.x * GRAM_THREADS) {
    double v[T];
#pragma unroll
    for (int k = 0; k < T; ++k) v[k] = (double)__ldg(g + k * ld + c);
    int p = 0;
#pragma unroll
    for (int i = 0; i < T; ++i)
#pragma unroll
      for (int j = i; j < T; ++j) acc[p] = fma(v[i], v[j], acc[p]), ++p;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int p = 0; p < NP; ++p) {
    const double v = warp_sum_d(acc[p]);
    if (lane == 0) s[warp][p] = v;
  }
  __syncthreads();
  if (threadIdx.x < NP) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < GRAM_THREADS / 32; ++w) v += s[w][threadIdx.x];
    partial[(int64_t)blockIdx.x * NP + threadIdx.x] = v;
  }
}

// Stage 2: one CTA; warp w adds the G partials of pairs w, w + 8, ... (lane-strided, then a shuffle tree) and writes both
// triangles of gram.
__global__ void __launch_bounds__(GRAM_THREADS)
gram_finish_kernel(const double* __restrict__ partial, int G, int T, double* __restrict__ gram) {
  const int NP = num_pairs(T);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int p = warp; p < NP; p += GRAM_THREADS / 32) {
    double v = 0.0;
    for (int k = lane; k < G; k += 32) v += partial[(int64_t)k * NP + p];
    v = warp_sum_d(v);
    if (lane == 0) {
      int i = 0, q = p;
      while (q >= T - i) q -= T - i, ++i;
      const int j = i + q;
      gram[i * T + j] = v;
      gram[j * T + i] = v;
    }
  }
}

// PCGrad in coefficient space, then out = sum_k c_k g_k.  Thread i < T of every CTA projects row i of C (g_i' = sum_k
// C[i][k] g_k) against the tasks in `order`; thread k then sums column k.  The stream accumulates in float64, so T = 1 and
// exact cancellations (antiparallel rows) come out exact.
template <int T>
__global__ void __launch_bounds__(COMBINE_THREADS)
pcgrad_combine_kernel(const float* __restrict__ g, int64_t ld, int64_t P, const double* __restrict__ gram,
                      const int* __restrict__ order, float* __restrict__ out, double* __restrict__ coef) {
  __shared__ double s_gram[T * T];
  __shared__ double s_C[T][T];
  __shared__ double s_c[T];
  __shared__ int s_order[T];
  if (threadIdx.x < T * T) s_gram[threadIdx.x] = gram[threadIdx.x];
  if (threadIdx.x < T) s_order[threadIdx.x] = order[threadIdx.x];
  __syncthreads();
  if (threadIdx.x < T) {
    const int i = threadIdx.x;
    for (int k = 0; k < T; ++k) s_C[i][k] = k == i ? 1.0 : 0.0;
    for (int n = 0; n < T; ++n) {
      const int j = s_order[n];
      if (j < 0 || j >= T || j == i) continue;          // not a permutation entry: ignored
      double dot = 0.0;
      for (int k = 0; k < T; ++k) dot = fma(s_C[i][k], s_gram[k * T + j], dot);
      const double gjj = s_gram[j * T + j];
      if (dot < 0.0 && gjj > 0.0) s_C[i][j] -= dot / gjj;
    }
  }
  __syncthreads();
  if (threadIdx.x < T) {
    const int k = threadIdx.x;
    double c = 0.0;
    for (int i = 0; i < T; ++i) c += s_C[i][k];
    s_c[k] = c;
    if (coef != nullptr && blockIdx.x == 0) coef[k] = c;
  }
  __syncthreads();
  double c[T];
#pragma unroll
  for (int k = 0; k < T; ++k) c[k] = s_c[k];
  for (int64_t col = (int64_t)blockIdx.x * COMBINE_THREADS + threadIdx.x; col < P;
       col += (int64_t)gridDim.x * COMBINE_THREADS) {
    double acc = c[0] * (double)__ldg(g + col);        // not fma(.., 0.0): keeps -0.0 at T = 1
#pragma unroll
    for (int k = 1; k < T; ++k) acc = fma(c[k], (double)__ldg(g + k * ld + col), acc);
    out[col] = (float)acc;
  }
}

// GradNorm (Chen et al. 2018, Algorithm 1) for T <= 8 tasks, one thread in float64.  The loops run over MAX_T with a
// T guard so that the per-task arrays stay in registers.
__global__ void gradnorm_update_kernel(const double* __restrict__ gram, const float* __restrict__ task_loss,
                                       const float* __restrict__ initial_loss, int T, float alpha, float lr,
                                       float* __restrict__ weights, float* __restrict__ grad_loss,
                                       float* __restrict__ d_weights) {
  if (threadIdx.x != 0) return;
  double n[MAX_T], G[MAX_T], q[MAX_T], w[MAX_T];
  double G_mean = 0.0, q_mean = 0.0;
#pragma unroll
  for (int t = 0; t < MAX_T; ++t) {
    if (t < T) {
      w[t] = (double)weights[t];
      n[t] = sqrt(gram[t * T + t]);
      G[t] = w[t] * n[t];
      q[t] = (double)task_loss[t] / (double)initial_loss[t];
      G_mean += G[t];
      q_mean += q[t];
    }
  }
  G_mean /= T;
  q_mean /= T;
  if (!(q_mean > 0.0)) {  // every current loss is 0 (B = 0, or a batch fitted exactly): r_t is 0/0, leave w as it is
#pragma unroll
    for (int t = 0; t < MAX_T; ++t)
      if (t < T && d_weights != nullptr) d_weights[t] = 0.f;
    grad_loss[0] = 0.f;
    return;
  }
  double L_grad = 0.0, w_sum = 0.0;
#pragma unroll
  for (int t = 0; t < MAX_T; ++t) {
    if (t < T) {
      const double diff = G[t] - G_mean * pow(q[t] / q_mean, (double)alpha);
      L_grad += fabs(diff);
      const double dw = (double)((diff > 0.0) - (diff < 0.0)) * n[t];
      if (d_weights != nullptr) d_weights[t] = (float)dw;
      w[t] -= (double)lr * dw;
      w_sum += w[t];
    }
  }
#pragma unroll
  for (int t = 0; t < MAX_T; ++t)
    if (t < T) weights[t] = (float)((double)T * w[t] / w_sum);
  grad_loss[0] = (float)L_grad;
}

static inline int gram_ctas(int64_t P) {
  return capped_grid((P + GRAM_COLS_PER_CTA - 1) / GRAM_COLS_PER_CTA, GRAM_MAX_CTAS);
}

}  // namespace mtl
}  // namespace ctr

using namespace ctr;
using namespace ctr::mtl;

#define MTL_CHECK_T(name, T) \
  CTR_UNSUPPORTED((T) < 1 || (T) > MAX_T, name ": T=%lld outside 1..8", (long long)(T))
#define MTL_CHECK_N(name, what, v) \
  CTR_UNSUPPORTED((v) < 0 || (v) > 0x7fffffffLL, name ": " what "=%lld outside 0..2^31-1", (long long)(v))

extern "C" int ctr_multitask_sigmoid_ce(const float* logits, const float* labels, int64_t T, int64_t B, int method,
                                        const float* task_param, float* task_loss, float* total_loss, float* d_logits,
                                        float* d_task_param, void* stream) {
  CTR_REQUIRE(logits && labels && task_loss && total_loss,
              "ctr_multitask_sigmoid_ce: null logits/labels/task_loss/total_loss");
  CTR_REQUIRE(method >= 0 && method <= 2, "ctr_multitask_sigmoid_ce: method=%d is not 0 (sum), 1 (weights) or 2 (uncertainty)",
              method);
  CTR_REQUIRE(method == 0 || task_param, "ctr_multitask_sigmoid_ce: null task_param for method %d", method);
  MTL_CHECK_T("ctr_multitask_sigmoid_ce", T);
  MTL_CHECK_N("ctr_multitask_sigmoid_ce", "B", B);
  return launch("ctr_multitask_sigmoid_ce", multitask_ce_kernel, CE_CTAS, CE_THREADS, 0, as_stream(stream), logits, labels,
                (int)T, (int)B, method, task_param, task_loss, total_loss, d_logits, d_task_param);
}

extern "C" int ctr_multitask_gram_workspace_bytes(int64_t T, int64_t P, int64_t* bytes) {
  CTR_REQUIRE(bytes, "ctr_multitask_gram_workspace_bytes: null bytes");
  MTL_CHECK_T("ctr_multitask_gram_workspace_bytes", T);
  MTL_CHECK_N("ctr_multitask_gram_workspace_bytes", "P", P);
  *bytes = (int64_t)gram_ctas(P) * num_pairs((int)T) * (int64_t)sizeof(double);
  return CTR_OK;
}

extern "C" int ctr_multitask_gram(const float* grads, int64_t T, int64_t P, int64_t ld, double* gram, void* workspace,
                                  int64_t workspace_bytes, void* stream) {
  CTR_REQUIRE(grads && gram && workspace, "ctr_multitask_gram: null grads/gram/workspace");
  MTL_CHECK_T("ctr_multitask_gram", T);
  MTL_CHECK_N("ctr_multitask_gram", "P", P);
  CTR_REQUIRE(ld >= P, "ctr_multitask_gram: ld=%lld < P=%lld", (long long)ld, (long long)P);
  const int G = gram_ctas(P);
  const int64_t need = (int64_t)G * num_pairs((int)T) * (int64_t)sizeof(double);
  CTR_REQUIRE(workspace_bytes >= need, "ctr_multitask_gram: workspace of %lld bytes, need %lld", (long long)workspace_bytes,
              (long long)need);
  cudaStream_t st = as_stream(stream);
  double* partial = static_cast<double*>(workspace);
  if (G > 0) {
    const int rc = with_const<1, 2, 3, 4, 5, 6, 7, 8>((int)T, [&](auto tc) {
      return launch("ctr_multitask_gram", gram_partial_kernel<decltype(tc)::value>, G, GRAM_THREADS, 0, st, grads, ld, P,
                    partial);
    });
    if (rc != CTR_OK) return rc;
  }
  return launch("ctr_multitask_gram", gram_finish_kernel, 1, GRAM_THREADS, 0, st, (const double*)partial, G, (int)T, gram);
}

extern "C" int ctr_pcgrad_combine(const float* grads, int64_t T, int64_t P, int64_t ld, const double* gram,
                                  const int32_t* order, float* out, double* coef, void* stream) {
  CTR_REQUIRE(grads && gram && order && out, "ctr_pcgrad_combine: null grads/gram/order/out");
  MTL_CHECK_T("ctr_pcgrad_combine", T);
  MTL_CHECK_N("ctr_pcgrad_combine", "P", P);
  CTR_REQUIRE(ld >= P, "ctr_pcgrad_combine: ld=%lld < P=%lld", (long long)ld, (long long)P);
  // at least one CTA, so that coef is written at P = 0
  const int grid = capped_grid(P > 0 ? (P + COMBINE_THREADS * 4 - 1) / (COMBINE_THREADS * 4) : 1, (int64_t)sm_count() * 4);
  return with_const<1, 2, 3, 4, 5, 6, 7, 8>((int)T, [&](auto tc) {
    return launch("ctr_pcgrad_combine", pcgrad_combine_kernel<decltype(tc)::value>, grid, COMBINE_THREADS, 0,
                  as_stream(stream), grads, ld, P, gram, (const int*)order, out, coef);
  });
}

extern "C" int ctr_gradnorm_update(const double* gram, const float* task_loss, const float* initial_loss, int64_t T,
                                   float alpha, float lr, float* weights, float* grad_loss, float* d_weights, void* stream) {
  CTR_REQUIRE(gram && task_loss && initial_loss && weights && grad_loss,
              "ctr_gradnorm_update: null gram/task_loss/initial_loss/weights/grad_loss");
  MTL_CHECK_T("ctr_gradnorm_update", T);
  return launch("ctr_gradnorm_update", gradnorm_update_kernel, 1, 32, 0, as_stream(stream), gram, task_loss, initial_loss,
                (int)T, alpha, lr, weights, grad_loss, d_weights);
}

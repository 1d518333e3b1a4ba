// Wide & Deep wide part (WideAndDeep/wide_and_deep.py:121-122,208-210,254-257): a hashed crossed column behind an indicator
// column, a dense(1) layer over the (B, num_buckets) multi-hot, and FTRL-Proximal on its variables.
//
// Reference: crossed_column([userid, manual_tag_list], hash_bucket_size=100000) -> indicator_column -> fc.input_layer ->
// tf.layers.dense(wide_input, 1) under wide_part, trained by tf.train.FtrlOptimizer.  [TF-internal, SURVEY A.11] the cross
// hashes the keys' vocabulary ids (int64, OOV -1 included) of every element of the Cartesian product of the keys' values,
// last key fastest:
//     h = hash_key (0xDECAFCAFFE); for each key k: h = FingerprintCat64(h, (uint64) v_k);   id = h % num_buckets
// The multi-hot counts duplicates, so wide_logit[b] = bias + sum over b's crosses of kernel[id].  Its kernel gradient is the
// DENSE multi_hot^T d_logit, so TF applies dense ApplyFtrl [TF-internal, SURVEY A.12] to both variables.
//
// H100 mapping (CUDA cores, no tensor-core work):
//   ctr_crossed_indicator_fwd  one warp per sample: lanes stride over the product index (decoded in mixed radix), hash,
//                              gather the kernel entry and warp-reduce; the crossed ids never reach memory.  Gather bound.
//   ctr_crossed_indicator_bwd  memset d_kernel, then the same enumeration scatter-adds d_logit[b] per cross.
//   ctr_ftrl_apply             one grid-stride 128-bit streaming pass over var, accum, linear and grad.  HBM bound.
#include "ctr_common.cuh"

namespace ctr {

__device__ __forceinline__ unsigned long long shift_mix(unsigned long long x) { return x ^ (x >> 47); }

// FingerprintCat64 of TF's core/platform/fingerprint.h
__device__ __forceinline__ unsigned long long fingerprint_cat64(unsigned long long a, unsigned long long b) {
  constexpr unsigned long long kMul = 0xc6a4a7935bd1e995ULL;
  unsigned long long r = a ^ kMul;
  r ^= shift_mix(b * kMul) * kMul;
  r *= kMul;
  r = shift_mix(r) * kMul;
  return shift_mix(r);
}

// The crosses of sample b: lo[k], n[k] locate key k's values; returns the number of crosses (0 if any key is empty).
struct SampleKeys {
  long long lo[4], n[4];
  long long count;
};
template <int K>
__device__ __forceinline__ SampleKeys sample_keys(const long long* __restrict__ offsets, int B, int b) {
  SampleKeys s;
  s.count = 1;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    s.lo[k] = __ldg(offsets + (size_t)k * (B + 1) + b);
    s.n[k] = __ldg(offsets + (size_t)k * (B + 1) + b + 1) - s.lo[k];
    s.count *= s.n[k] > 0 ? s.n[k] : 0;
  }
  return s;
}
// Bucket of cross p (mixed radix, last key fastest).
template <int K>
__device__ __forceinline__ long long cross_bucket(const long long* __restrict__ values, const SampleKeys& s, long long p,
                                                  unsigned long long hash_key, unsigned long long num_buckets) {
  long long idx[K];
#pragma unroll
  for (int k = K - 1; k >= 0; --k) {
    idx[k] = p % s.n[k];
    p /= s.n[k];
  }
  unsigned long long h = hash_key;
#pragma unroll
  for (int k = 0; k < K; ++k) h = fingerprint_cat64(h, (unsigned long long)__ldg(values + s.lo[k] + idx[k]));
  return (long long)(h % num_buckets);
}

template <int K>
__global__ void __launch_bounds__(256)
crossed_indicator_fwd_kernel(const long long* __restrict__ values, const long long* __restrict__ offsets, int B,
                             unsigned long long num_buckets, unsigned long long hash_key, const float* __restrict__ kernel,
                             const float* __restrict__ bias, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const float b0 = __ldg(bias);
  for (int b = warp0; b < B; b += nwarps) {
    const SampleKeys s = sample_keys<K>(offsets, B, b);
    float acc = 0.f;
    for (long long p = lane; p < s.count; p += 32) acc += __ldg(kernel + cross_bucket<K>(values, s, p, hash_key, num_buckets));
    acc = warp_sum(acc);
    if (lane == 0) out[b] = acc + b0;
  }
}

template <int K>
__global__ void __launch_bounds__(256)
crossed_indicator_bwd_kernel(const long long* __restrict__ values, const long long* __restrict__ offsets, int B,
                             unsigned long long num_buckets, unsigned long long hash_key, const float* __restrict__ d_logit,
                             float* __restrict__ d_kernel, float* __restrict__ d_bias) {
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  float gsum = 0.f;
  for (int b = warp0; b < B; b += nwarps) {
    const SampleKeys s = sample_keys<K>(offsets, B, b);
    const float g = __ldg(d_logit + b);
    gsum += g;
    for (long long p = lane; p < s.count; p += 32) atomicAdd(d_kernel + cross_bucket<K>(values, s, p, hash_key, num_buckets), g);
  }
  if (d_bias != nullptr && lane == 0 && warp0 < B) atomicAdd(d_bias, gsum);
}

// TF's ApplyFtrl functor (core/kernels/training_ops.cc), one element; l2x2 = 2 * l2.
template <bool SQRT>
__device__ __forceinline__ void ftrl_elem(float& var, float& accum, float& linear, float g, float lr, float lr_power, float l1,
                                          float l2x2) {
  const float new_accum = accum + g * g;
  const float pn = SQRT ? sqrtf(new_accum) : powf(new_accum, -lr_power);
  const float po = SQRT ? sqrtf(accum) : powf(accum, -lr_power);
  linear += g - (pn - po) / lr * var;
  const float sgn = linear > 0.f ? 1.f : (linear < 0.f ? -1.f : 0.f);
  const float x = l1 * sgn - linear;
  const float y = pn / lr + l2x2;
  var = fabsf(linear) > l1 ? x / y : 0.f;
  accum = new_accum;
}

// head: elements before the first 16-byte boundary of the four buffers when they share it (vec), handled one per thread
// like the tail; buffers that do not share it (!vec) take the scalar grid-stride loop.
template <bool SQRT>
__global__ void __launch_bounds__(256)
ftrl_apply_kernel(float* __restrict__ var, float* __restrict__ accum, float* __restrict__ linear, const float* __restrict__ grad,
                  long long n, int head, bool vec, float lr, float lr_power, float l1, float l2x2) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  auto scalar = [&](long long i) {
    float w = var[i], a = accum[i], l = linear[i];
    ftrl_elem<SQRT>(w, a, l, grad[i], lr, lr_power, l1, l2x2);
    var[i] = w; accum[i] = a; linear[i] = l;
  };
  if (!vec) {
    for (long long i = t0; i < n; i += stride) scalar(i);
    return;
  }
  if (t0 < head) scalar(t0);
  const long long n4 = (n - head) / 4;
  auto* v4 = reinterpret_cast<float4*>(var + head);
  auto* a4 = reinterpret_cast<float4*>(accum + head);
  auto* l4 = reinterpret_cast<float4*>(linear + head);
  const auto* g4 = reinterpret_cast<const float4*>(grad + head);
  for (long long i = t0; i < n4; i += stride) {
    float4 w = ldg_stream_f4(v4 + i), a = ldg_stream_f4(a4 + i), l = ldg_stream_f4(l4 + i);
    const float4 g = ldg_stream_f4(g4 + i);
    ftrl_elem<SQRT>(w.x, a.x, l.x, g.x, lr, lr_power, l1, l2x2);
    ftrl_elem<SQRT>(w.y, a.y, l.y, g.y, lr, lr_power, l1, l2x2);
    ftrl_elem<SQRT>(w.z, a.z, l.z, g.z, lr, lr_power, l1, l2x2);
    ftrl_elem<SQRT>(w.w, a.w, l.w, g.w, lr, lr_power, l1, l2x2);
    stg_stream_f4(v4 + i, w); stg_stream_f4(a4 + i, a); stg_stream_f4(l4 + i, l);
  }
  const long long tail = head + n4 * 4 + t0;                 // the last (n - head) % 4 elements, one per thread
  if (tail < n) scalar(tail);
}

static int check_cross(const char* fn, int64_t K, int64_t B, int64_t num_buckets) {
  CTR_REQUIRE(B >= 0 && B <= 0x7fffffffLL / 8, "%s: bad B=%lld", fn, (long long)B);
  CTR_UNSUPPORTED(K < 2 || K > 4, "%s: K=%lld keys unsupported (2 <= K <= 4)", fn, (long long)K);
  CTR_UNSUPPORTED(num_buckets < 2 || num_buckets >= (1LL << 31), "%s: num_buckets=%lld unsupported (2 <= num_buckets < 2^31)", fn,
                  (long long)num_buckets);
  return CTR_OK;
}

static int cross_grid(int64_t B) { return capped_grid((B + 7) / 8, (long long)sm_count() * 8); }

}  // namespace ctr

using namespace ctr;

extern "C" int ctr_crossed_indicator_fwd(const int64_t* values, const int64_t* offsets, int64_t K, int64_t B, int64_t num_buckets,
                                         uint64_t hash_key, const float* kernel, const float* bias, float* out, void* stream) {
  const char* fn = "ctr_crossed_indicator_fwd";
  CTR_REQUIRE(values && offsets && kernel && bias && out, "%s: null argument", fn);
  int rc = check_cross(fn, K, B, num_buckets);
  if (rc || B == 0) return rc;
  return with_const<2, 3, 4>((int)K, [&](auto KK) {
    return launch(fn, crossed_indicator_fwd_kernel<KK>, cross_grid(B), 256, 0, as_stream(stream), reinterpret_cast<const long long*>(values),
                  reinterpret_cast<const long long*>(offsets), (int)B, (unsigned long long)num_buckets, (unsigned long long)hash_key,
                  kernel, bias, out);
  });
}

extern "C" int ctr_crossed_indicator_bwd(const int64_t* values, const int64_t* offsets, int64_t K, int64_t B, int64_t num_buckets,
                                         uint64_t hash_key, const float* d_logit, float* d_kernel, float* d_bias, void* stream) {
  const char* fn = "ctr_crossed_indicator_bwd";
  CTR_REQUIRE(values && offsets && d_logit && d_kernel, "%s: null argument", fn);
  int rc = check_cross(fn, K, B, num_buckets);
  if (rc) return rc;
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(d_kernel, 0, (size_t)num_buckets * sizeof(float), st));
  if (d_bias != nullptr) CTR_CUDA(cudaMemsetAsync(d_bias, 0, sizeof(float), st));
  if (B == 0) return CTR_OK;
  return with_const<2, 3, 4>((int)K, [&](auto KK) {
    return launch(fn, crossed_indicator_bwd_kernel<KK>, cross_grid(B), 256, 0, st, reinterpret_cast<const long long*>(values),
                  reinterpret_cast<const long long*>(offsets), (int)B, (unsigned long long)num_buckets, (unsigned long long)hash_key,
                  d_logit, d_kernel, d_bias);
  });
}

extern "C" int ctr_ftrl_apply(float* var, float* accum, float* linear, const float* grad, int64_t n, float lr, float lr_power,
                              float l1, float l2, void* stream) {
  const char* fn = "ctr_ftrl_apply";
  CTR_REQUIRE(var && accum && linear && grad, "%s: null argument", fn);
  CTR_REQUIRE(n >= 0, "%s: bad n=%lld", fn, (long long)n);
  CTR_REQUIRE(lr > 0.f, "%s: learning rate must be > 0", fn);
  CTR_REQUIRE(lr_power <= 0.f, "%s: lr_power must be <= 0", fn);
  CTR_REQUIRE(l1 >= 0.f && l2 >= 0.f, "%s: l1 and l2 must be >= 0", fn);
  auto phase = [](const void* p) { return reinterpret_cast<uintptr_t>(p) & 15u; };
  CTR_REQUIRE((phase(var) | phase(accum) | phase(linear) | phase(grad)) % 4 == 0, "%s: buffers must be 4-byte aligned floats", fn);
  if (n == 0) return CTR_OK;
  const bool vec = phase(var) == phase(accum) && phase(var) == phase(linear) && phase(var) == phase(grad);
  const long long head = vec ? (long long)((16 - phase(var)) % 16 / 4) : 0;
  const int h = (int)(head < n ? head : n);
  const int grid = capped_grid(((vec ? (n - h) / 4 : n) + 255) / 256 + 1, (long long)sm_count() * 16);
  auto go = [&](auto k) {
    return launch(fn, k, grid, 256, 0, as_stream(stream), var, accum, linear, grad, (long long)n, h, vec, lr, lr_power, l1, 2.f * l2);
  };
  return lr_power == -0.5f ? go(ftrl_apply_kernel<true>) : go(ftrl_apply_kernel<false>);
}

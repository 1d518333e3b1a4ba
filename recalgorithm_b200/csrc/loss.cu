// The last step of the e2e path: mean sigmoid cross-entropy of the summed logits and its gradient, one launch.
//
// Reference: loss = tf.reduce_mean(tf.nn.sigmoid_cross_entropy_with_logits(labels=y, logits=logits)) with
// logits = add_n([first_order, fm2, deep]) -- DeepFM/deepfm.py:214,235 (same line in every model_fn); TF's stable form
// (SURVEY A.7):  l = max(x,0) - x*z + log1p(exp(-|x|)),   dl/dx = sigmoid(x) - z.
// Not part of the hot path's arithmetic (the dense tail is out of scope); it exists so that the public-API step
// (bench.py e2e) is not a dozen 3-microsecond elementwise launches around two 0.1 ms kernels.
#include "ctr_common.cuh"

namespace ctr {

__global__ void __launch_bounds__(256)
sigmoid_ce_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ labels, int B, float inv_b,
                  float* __restrict__ loss, float* __restrict__ d_logit) {
  float acc = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
    const float x = __ldg(a + i) + (b ? __ldg(b + i) : 0.f);
    const float z = __ldg(labels + i);
    acc += fmaxf(x, 0.f) - x * z + log1pf(expf(-fabsf(x)));
    if (d_logit != nullptr) d_logit[i] = (1.f / (1.f + expf(-x)) - z) * inv_b;
  }
  acc = warp_sum(acc);
  __shared__ float s[8];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 8) {
    float v = s[threadIdx.x];
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(0xffu, v, o);
    if (threadIdx.x == 0) atomicAdd(loss, v * inv_b);
  }
}

}  // namespace ctr

using namespace ctr;

extern "C" int ctr_sigmoid_ce(const float* logit_a, const float* logit_b, const float* labels, int64_t B, float* loss,
                              float* d_logit, void* stream) {
  CTR_REQUIRE(logit_a && labels && loss, "ctr_sigmoid_ce: null logit_a/labels/loss");
  CTR_REQUIRE(B >= 0 && B <= 0x7fffffffLL, "ctr_sigmoid_ce: bad B");
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), st));
  if (B == 0) return CTR_OK;
  return launch("ctr_sigmoid_ce", sigmoid_ce_kernel, capped_grid((B + 255) / 256, (int64_t)sm_count() * 2), 256, 0, st, logit_a,
                logit_b, labels, (int)B, 1.f / (float)B, loss, d_logit);
}

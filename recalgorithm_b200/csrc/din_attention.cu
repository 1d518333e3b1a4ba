// Row DIN-ATT (SURVEY.md section 8a): the DIN attention unit over the behaviour sequence.
//
// Reference: din_attention(query, keys, keys_length, is_softmax) -- DIN/din_attention.py:17-43
//   cross = [q, k, q-k, q*k] (4H) -> dense 64 relu (f1_att) -> dense 32 relu (f2_att) -> dense 1 (f3_att);
//   mask by sequence_mask(keys_length, T); default: weights*mask; softmax variant: fill -2**32+1, THEN /sqrt(H),
//   softmax over T; out = weights^T . keys  (B,H).
//
// H100 mapping (FP32-FMA-bound, CUDA cores; north_star keeps tensor cores for CIN only):
//   * one warp per sample; the sample's keys (T x H) are staged once in shared memory;
//   * layer 1 is algebraically folded per sample:  cross@W1 = q@(W1a+W1c) + k@(W1b-W1c) + (q*k)@W1d
//       = qpart + k @ Weff,  Weff[h,c] = (W1b-W1c)[h,c] + q[h]*W1d[h,c]   (H x 64 per sample, in registers)
//     so the q side is hoisted out of the T loop and layer 1 costs H*64 instead of 4H*64 MACs per position;
//   * lane c owns output column c of each dense layer; activations of the previous layer are broadcast from
//     shared memory with 128-bit loads; W2's column lives in 64 registers;
//   * positions t >= keys_length never reach the MLP: their weight is exactly 0 (or the constant pad) in the
//     reference, so the result is identical and ~half the FLOPs disappear for uniformly distributed lengths;
//   * backward recomputes the MLP per position (nothing but the (B,T) weights is saved), produces input
//     gradients per warp, and reduces the weight gradients CTA-cooperatively with thread-owned register
//     accumulators (rank-k updates over the positions staged by all warps), merged by fp32 atomics.
#include <math.h>

#include "ctr_common.cuh"

namespace ctr {

constexpr int DIN_H1 = 64;      // f1_att units (DIN/din_attention.py:21)
constexpr int DIN_H2 = 32;      // f2_att units (:22)
constexpr int DIN_TT = 4;       // positions per warp per round
constexpr int DIN_BT = 2;       // backward: positions per warp per round (4 measured no faster: the unrolled body outgrew the
                                // 32 KB instruction cache -- 23 % of the stall samples were instruction fetches)
constexpr int DIN_SCHED_HDR = 64;   // ints in front of the order array of the schedule scratch ([0] = work counter)
constexpr float DIN_PAD_F = -4294967295.0f;   // -2**32 + 1 (rounds to -2^32 in fp32, like the reference's fp32 tensor)

struct DinSmem {                // offsets in floats into dynamic shared memory
  int wq, wk, wd, b1, w2, b2, w3, w1t, per_warp, warp_stride, tile, tile_stride, total;
};
// offsets inside one staged position of the backward tile
__host__ __device__ inline int din_off_cross() { return DIN_H1; }
__host__ __device__ inline int din_off_dpre1(int H) { return DIN_H1 + 4 * H; }
__host__ __device__ inline int din_off_h2(int H) { return 2 * DIN_H1 + 4 * H; }
__host__ __device__ inline int din_off_dpre2(int H) { return 2 * DIN_H1 + DIN_H2 + 4 * H; }
__host__ __device__ inline int din_off_dcross(int H) { return 2 * DIN_H1 + 2 * DIN_H2 + 4 * H; }
__host__ __device__ inline int din_off_ds(int H) { return 2 * DIN_H1 + 2 * DIN_H2 + 8 * H; }

__host__ __device__ inline DinSmem din_layout(int H, int T, int warps, bool bwd) {
  DinSmem L;
  int o = 0;
  L.wq = o; o += H * DIN_H1;                      // (H,64)  W1a + W1c
  L.wk = o; o += H * DIN_H1;                      // (H,64)  W1b - W1c
  L.wd = o; o += H * DIN_H1;                      // (H,64)  W1d
  L.b1 = o; o += DIN_H1;
  L.w2 = o; o += DIN_H1 * DIN_H2;                 // (64,32) row-major (bwd reads rows; fwd loads columns to registers)
  L.b2 = o; o += DIN_H2;
  L.w3 = o; o += DIN_H2 + 4;                      // w3 (32) + b3 (1), padded
  L.w1t = o; o += bwd ? DIN_H1 * 4 * H : 0;       // (64, 4H) = W1 transposed, for dcross = dpre1 @ W1^T
  L.per_warp = o;
  // per warp: keys (T*H) | sc (T) | q (H) | go (H) | dq (H)  (+ bwd: dkeys (T*H), ds (T))
  int ws = T * H + T + 3 * H + (bwd ? T * H + T : 0);
  ws = (ws + 3) & ~3;
  L.warp_stride = ws;
  o += warps * ws;
  L.tile = o;
  // per warp, per staged position: h1 (64) | [bwd: cross (4H) | dpre1 (64) | h2 (32) | dpre2 (32) | dcross (4H) | ds (4)]
  int ts = DIN_H1 + (bwd ? 4 * H + DIN_H1 + DIN_H2 + DIN_H2 + 4 * H + 4 : 0);
  L.tile_stride = ts;
  o += warps * DIN_TT * ts;
  L.total = o;
  return L;
}

__device__ __forceinline__ void din_stage_weights(float* sm, const DinSmem& L, const float* __restrict__ w1,
                                                  const float* __restrict__ b1, const float* __restrict__ w2,
                                                  const float* __restrict__ b2, const float* __restrict__ w3,
                                                  const float* __restrict__ b3, int H, bool bwd) {
  for (int i = threadIdx.x; i < H * DIN_H1; i += blockDim.x) {
    const float a = __ldg(w1 + i), b = __ldg(w1 + H * DIN_H1 + i), c = __ldg(w1 + 2 * H * DIN_H1 + i),
                d = __ldg(w1 + 3 * H * DIN_H1 + i);
    sm[L.wq + i] = a + c;
    sm[L.wk + i] = b - c;
    sm[L.wd + i] = d;
  }
  for (int i = threadIdx.x; i < DIN_H1; i += blockDim.x) sm[L.b1 + i] = __ldg(b1 + i);
  for (int i = threadIdx.x; i < DIN_H1 * DIN_H2; i += blockDim.x) sm[L.w2 + i] = __ldg(w2 + i);
  for (int i = threadIdx.x; i < DIN_H2; i += blockDim.x) { sm[L.b2 + i] = __ldg(b2 + i); sm[L.w3 + i] = __ldg(w3 + i); }
  if (threadIdx.x == 0) sm[L.w3 + DIN_H2] = __ldg(b3);
  if (bwd)
    for (int i = threadIdx.x; i < 4 * H * DIN_H1; i += blockDim.x) {
      const int r = i / DIN_H1, c = i % DIN_H1;                     // w1[r][c] -> w1t[c][r]
      sm[L.w1t + c * 4 * H + r] = __ldg(w1 + i);
    }
}

// Per-sample preparation shared by fwd and bwd: stage keys + q, fold layer 1.
template <int HP>
__device__ __forceinline__ void din_prepare(float* sm, const DinSmem& L, float* wsm, const float* __restrict__ query,
                                            const float* __restrict__ keys, int b, int T, int H, int lane,
                                            float (&weff)[HP][2], float (&qpart)[2]) {
  float* skeys = wsm;
  float* sq = wsm + T * H + T;
  for (int i = lane; i < T * H; i += 32) skeys[i] = __ldg(keys + (size_t)b * T * H + i);
  for (int i = lane; i < H; i += 32) sq[i] = __ldg(query + (size_t)b * H + i);
  __syncwarp();
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int c = lane + 32 * u;
    float acc = sm[L.b1 + c];
#pragma unroll
    for (int h = 0; h < HP; ++h) {
      if (h < H) {
        const float qh = sq[h];
        acc += qh * sm[L.wq + h * DIN_H1 + c];
        weff[h][u] = sm[L.wk + h * DIN_H1 + c] + qh * sm[L.wd + h * DIN_H1 + c];
      } else {
        weff[h][u] = 0.f;
      }
    }
    qpart[u] = acc;
  }
}

// Forward MLP for up to DIN_TT positions t0..t0+n-1 of the staged sample.  Writes h1 to the warp's tile area and
// returns (lane-owned) h2 and the scores.
template <int HP>
__device__ __forceinline__ void din_mlp_tile(const float* sm, const DinSmem& L, const float* skeys, float* tile,
                                             int t0, int n, int H, int lane, const float (&weff)[HP][2],
                                             const float (&qpart)[2], const float (&w2col)[DIN_H1],
                                             float (&h2)[DIN_TT], float (&score)[DIN_TT]) {
#pragma unroll
  for (int tt = 0; tt < DIN_TT; ++tt) {
    if (tt < n) {
      const float* k = skeys + (t0 + tt) * H;
      float p0 = qpart[0], p1 = qpart[1];
#pragma unroll
      for (int h = 0; h < HP; ++h) {
        if (h < H) {
          const float kv = k[h];
          p0 += kv * weff[h][0];
          p1 += kv * weff[h][1];
        }
      }
      tile[tt * L.tile_stride + lane] = fmaxf(p0, 0.f);
      tile[tt * L.tile_stride + lane + 32] = fmaxf(p1, 0.f);
    }
  }
  __syncwarp();
  const float b2v = sm[L.b2 + lane], w3v = sm[L.w3 + lane], b3v = sm[L.w3 + DIN_H2];
#pragma unroll
  for (int tt = 0; tt < DIN_TT; ++tt) {
    h2[tt] = 0.f;
    score[tt] = 0.f;
    if (tt < n) {
      const float4* h1v = reinterpret_cast<const float4*>(tile + tt * L.tile_stride);
      float acc = b2v;
#pragma unroll
      for (int c4 = 0; c4 < DIN_H1 / 4; ++c4) {
        const float4 v = h1v[c4];
        acc += v.x * w2col[4 * c4 + 0];
        acc += v.y * w2col[4 * c4 + 1];
        acc += v.z * w2col[4 * c4 + 2];
        acc += v.w * w2col[4 * c4 + 3];
      }
      h2[tt] = fmaxf(acc, 0.f);
      score[tt] = warp_sum(h2[tt] * w3v) + b3v;
    }
  }
}

// scores (smem, first `len` valid) -> attention weights in place, following DIN/din_attention.py:27-38.
__device__ __forceinline__ void din_weights(float* sc, int T, int len, int H, int is_softmax, int lane) {
  if (!is_softmax) {
    for (int t = lane; t < T; t += 32) sc[t] = t < len ? sc[t] : 0.f;        // weights * mask
  } else {
    const float scale = sqrtf((float)H);
    float m = -INFINITY;
    for (int t = lane; t < T; t += 32) {
      const float v = (t < len ? sc[t] : DIN_PAD_F) / scale;                 // where(mask, w, pad) THEN / sqrt(H)
      sc[t] = v;
      m = fmaxf(m, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int t = lane; t < T; t += 32) {
      const float e = expf(sc[t] - m);
      sc[t] = e;
      s += e;
    }
    s = warp_sum(s);
    for (int t = lane; t < T; t += 32) sc[t] = sc[t] / s;
  }
  __syncwarp();
}

// Work distribution.  A warp's cost is its samples' keys_length (0..T), so a static round-robin leaves the CTA waiting for
// its slowest warp (ncu: 26 % of the backward's stall samples at the final barrier, and SMs idle behind it).  One tiny
// kernel counting-sorts the sample ids by DESCENDING length into sched[64 + i]; warps then take samples from a global counter
// (sched[0]) -- longest-processing-time-first list scheduling.  sched == NULL keeps the static assignment.
__global__ void __launch_bounds__(1024)
din_schedule_kernel(const long long* __restrict__ keys_length, int B, int T, int* __restrict__ sched) {
  extern __shared__ int s_bin[];                       // (T + 2) bins, then their start offsets
  for (int i = threadIdx.x; i < T + 2; i += blockDim.x) s_bin[i] = 0;
  if (threadIdx.x == 0) sched[0] = 0;
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    long long l = __ldg(keys_length + b);
    const int len = (int)(l < 0 ? 0 : (l > T ? T : l));
    atomicAdd(&s_bin[T - len], 1);                     // bin 0 = longest
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int i = 0; i <= T; ++i) { const int c = s_bin[i]; s_bin[i] = acc; acc += c; }
  }
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    long long l = __ldg(keys_length + b);
    const int len = (int)(l < 0 ? 0 : (l > T ? T : l));
    sched[DIN_SCHED_HDR + atomicAdd(&s_bin[T - len], 1)] = b;
  }
}

// next sample of this warp: static stride, or the shared work counter over the longest-first order
__device__ __forceinline__ int din_next_sample(int* __restrict__ sched, int B, int& static_b, int stride, int lane) {
  if (sched == nullptr) {
    const int b = static_b;
    static_b += stride;
    return b < B ? b : -1;
  }
  int i = 0;
  if (lane == 0) i = atomicAdd(sched, 1);
  i = __shfl_sync(0xffffffffu, i, 0);
  return i < B ? __ldg(sched + DIN_SCHED_HDR + i) : -1;
}

template <int HP, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
din_attention_fwd_kernel(const float* __restrict__ query, const float* __restrict__ keys,
                         const long long* __restrict__ keys_length, const float* __restrict__ w1,
                         const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
                         const float* __restrict__ w3, const float* __restrict__ b3, int B, int T, int H,
                         int is_softmax, float* __restrict__ out, float* __restrict__ att_w, int* __restrict__ sched) {
  extern __shared__ __align__(16) float sm[];
  const DinSmem L = din_layout(H, T, WARPS, false);
  din_stage_weights(sm, L, w1, b1, w2, b2, w3, b3, H, false);
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float w2col[DIN_H1];
#pragma unroll
  for (int c = 0; c < DIN_H1; ++c) w2col[c] = sm[L.w2 + c * DIN_H2 + lane];
  float* wsm = sm + L.per_warp + wid * L.warp_stride;
  float* skeys = wsm;
  float* sc = wsm + T * H;
  float* tile = sm + L.tile + wid * DIN_TT * L.tile_stride;

  int static_b = blockIdx.x * WARPS + wid;
  for (int b = din_next_sample(sched, B, static_b, gridDim.x * WARPS, lane); b >= 0;
       b = din_next_sample(sched, B, static_b, gridDim.x * WARPS, lane)) {
    float weff[HP][2], qpart[2];
    __syncwarp();
    din_prepare<HP>(sm, L, wsm, query, keys, b, T, H, lane, weff, qpart);
    long long len64 = __ldg(keys_length + b);
    const int len = (int)(len64 < 0 ? 0 : (len64 > T ? T : len64));
    for (int t0 = 0; t0 < len; t0 += DIN_TT) {
      float h2[DIN_TT], score[DIN_TT];
      const int n = min(DIN_TT, len - t0);
      din_mlp_tile<HP>(sm, L, skeys, tile, t0, n, H, lane, weff, qpart, w2col, h2, score);
      if (lane == 0) {
#pragma unroll
        for (int tt = 0; tt < DIN_TT; ++tt)
          if (tt < n) sc[t0 + tt] = score[tt];
      }
      __syncwarp();
    }
    din_weights(sc, T, len, H, is_softmax, lane);
    for (int h = lane; h < H; h += 32) {
      float acc = 0.f;
      for (int t = 0; t < T; ++t) acc += sc[t] * skeys[t * H + h];           // matmul(w^T, keys)
      out[(size_t)b * H + h] = acc;
    }
    if (att_w != nullptr)
      for (int t = lane; t < T; t += 32) att_w[(size_t)b * T + t] = sc[t];
  }
}

// ---------------------------------------------------------------------------------------------------
// backward (second revision: every warp is independent -- no block-level phases)
// ---------------------------------------------------------------------------------------------------
// The first version staged per-position vectors for a CTA-cooperative rank-k update and needed two block syncs per
// 32 positions at one CTA (8 warps, 255 registers) per SM: 0.92 ms at config 4, issue slots 25 % used.  The weight
// gradient of layer 1 is restructured algebraically so that nothing per-position has to leave the warp:
//     D_b  = sum_t dpre1[t]            (64)         KD_b = sum_t k[t] (x) dpre1[t]      (H x 64, same shape as Weff)
//     dW1a = sum_b q_b (x) D_b         dW1b = sum_b KD_b       dW1c = dW1a - dW1b       dW1d = sum_b diag(q_b) KD_b
//     dq_b = (W1a+W1c) D_b + rowsum(W1d * KD_b)            dk[t] = Weff_b dpre1[t]
// so per position the warp only adds into 32 (KD) + 64 (dW2 column) + a few register accumulators; per SAMPLE it flushes
// 3*H*64 values into shared-memory accumulators; per CTA one set of global atomics at the end.
// d_params layout: [w1 (4H*64) | b1 (64) | w2 (64*32) | b2 (32) | w3 (32) | b3 (1)]
struct DinBwdSmem {
  int wq, wk, wd, b1, w2, b2, w3, aw2, ab2, aw3, per_warp, warp_stride, total;
  int o_sc, o_q, o_go, o_ds, o_acc, o_wt, o_h1, o_dp1, o_dp2;     // offsets inside a warp's region
};

__host__ __device__ inline DinBwdSmem din_bwd_layout(int H, int HP, int T, int warps) {
  DinBwdSmem L;
  int o = 0;
  L.wq = o; o += H * DIN_H1;
  L.wk = o; o += H * DIN_H1;
  L.wd = o; o += H * DIN_H1;
  L.b1 = o; o += DIN_H1;
  L.w2 = o; o += DIN_H1 * DIN_H2;
  L.b2 = o; o += DIN_H2;
  L.w3 = o; o += DIN_H2 + 4;
  L.aw2 = o; o += DIN_H1 * DIN_H2;
  L.ab2 = o; o += DIN_H2;
  L.aw3 = o; o += DIN_H2 + 4;                       // dw3 (32) + db3 (1)
  L.per_warp = o;
  int w = 0;
  w += T * H;                                       // keys
  L.o_sc = w; w += T;
  L.o_q = w; w += H;
  L.o_go = w; w += H;
  L.o_ds = w; w += T;
  w = (w + 3) & ~3;
  L.o_acc = w; w += 3 * H * DIN_H1 + DIN_H1;        // the WARP's private sums of dW1a | dW1b | dW1d | db1 over its samples (plain
                                                    // read-modify-writes: shared-memory atomics here cost 98 x 64 clk of the SM's
                                                    // atomic unit per sample = a third of the kernel)
  w = (w + 3) & ~3;
  L.o_wt = w; w += DIN_H1 * (HP + 1);               // Weff^T[c][h], padded rows
  w = (w + 3) & ~3;
  L.o_h1 = w; w += DIN_H1 * DIN_BT;
  L.o_dp1 = w; w += DIN_H1 * DIN_BT;
  L.o_dp2 = w; w += DIN_H2 * DIN_BT;
  w = (w + 3) & ~3;
  L.warp_stride = w;
  L.total = o + warps * w;
  return L;
}

template <int HP, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
din_attention_bwd_kernel(const float* __restrict__ query, const float* __restrict__ keys,
                         const long long* __restrict__ keys_length, const float* __restrict__ w1,
                         const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
                         const float* __restrict__ w3, const float* __restrict__ b3, const float* __restrict__ g_out,
                         const float* __restrict__ att_w, int B, int T, int H, int is_softmax,
                         float* __restrict__ d_query, float* __restrict__ d_keys, float* __restrict__ d_params,
                         int* __restrict__ sched) {
  extern __shared__ __align__(16) float sm[];
  const DinBwdSmem L = din_bwd_layout(H, HP, T, WARPS);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, tid = threadIdx.x;
  const int H4 = 4 * H;
  // ---- stage weights (folded like the forward) and zero the CTA accumulators
  for (int i = tid; i < H * DIN_H1; i += blockDim.x) {
    const float a = __ldg(w1 + i), b = __ldg(w1 + H * DIN_H1 + i), c = __ldg(w1 + 2 * H * DIN_H1 + i),
                d = __ldg(w1 + 3 * H * DIN_H1 + i);
    sm[L.wq + i] = a + c;
    sm[L.wk + i] = b - c;
    sm[L.wd + i] = d;
  }
  for (int i = tid; i < DIN_H1; i += blockDim.x) sm[L.b1 + i] = __ldg(b1 + i);
  for (int i = tid; i < DIN_H1 * DIN_H2; i += blockDim.x) { sm[L.w2 + i] = __ldg(w2 + i); sm[L.aw2 + i] = 0.f; }
  for (int i = tid; i < DIN_H2; i += blockDim.x) {
    sm[L.b2 + i] = __ldg(b2 + i); sm[L.w3 + i] = __ldg(w3 + i); sm[L.ab2 + i] = 0.f; sm[L.aw3 + i] = 0.f;
  }
  if (tid == 0) { sm[L.w3 + DIN_H2] = __ldg(b3); sm[L.aw3 + DIN_H2] = 0.f; }
  __syncthreads();

  float* wsm = sm + L.per_warp + wid * L.warp_stride;
  float* skeys = wsm;
  float* sc = wsm + L.o_sc;
  float* sq = wsm + L.o_q;
  float* sgo = wsm + L.o_go;
  float* sds = wsm + L.o_ds;
  float* pacc = wsm + L.o_acc;                 // [0,H*64) dW1a | [H*64, 2H*64) dW1b | [2H*64, 3H*64) dW1d | 64 db1
  for (int i = lane; i < 3 * H * DIN_H1 + DIN_H1; i += 32) pacc[i] = 0.f;
  __syncwarp();
  float* swt = wsm + L.o_wt;
  float* sh1 = wsm + L.o_h1;
  float* sdp1 = wsm + L.o_dp1;
  float* sdp2 = wsm + L.o_dp2;
  const float b2v = sm[L.b2 + lane], w3v = sm[L.w3 + lane], b3v = sm[L.w3 + DIN_H2];
  const float* W2s = sm + L.w2;

  // register accumulators that live for the whole kernel
  float acc_w2[DIN_H1];                         // column `lane` of dW2
#pragma unroll
  for (int c = 0; c < DIN_H1; ++c) acc_w2[c] = 0.f;
  float acc_b2 = 0.f, acc_w3 = 0.f, acc_b3 = 0.f;

  // layer-1 + layer-2 forward of one position from the folded per-sample weights; h1 goes to smem, returns h2 and score
  auto mlp_fwd = [&](const float* k, const float (&weff)[HP][2], const float (&qpart)[2], float& h1a, float& h1b,
                     float& h2, float& score) {
    float p0 = qpart[0], p1 = qpart[1];
#pragma unroll
    for (int h = 0; h < HP; ++h) {
      if (h < H) {
        const float kv = k[h];
        p0 += kv * weff[h][0];
        p1 += kv * weff[h][1];
      }
    }
    h1a = fmaxf(p0, 0.f); h1b = fmaxf(p1, 0.f);
    sh1[lane] = h1a; sh1[lane + 32] = h1b;
    __syncwarp();
    float acc = b2v;
    const float4* h1v = reinterpret_cast<const float4*>(sh1);
#pragma unroll
    for (int c4 = 0; c4 < DIN_H1 / 4; ++c4) {
      const float4 v = h1v[c4];
      acc += v.x * W2s[(4 * c4 + 0) * DIN_H2 + lane];
      acc += v.y * W2s[(4 * c4 + 1) * DIN_H2 + lane];
      acc += v.z * W2s[(4 * c4 + 2) * DIN_H2 + lane];
      acc += v.w * W2s[(4 * c4 + 3) * DIN_H2 + lane];
    }
    h2 = fmaxf(acc, 0.f);
    score = warp_sum(h2 * w3v) + b3v;
  };

  int static_b = blockIdx.x * WARPS + wid;
  for (int b = din_next_sample(sched, B, static_b, gridDim.x * WARPS, lane); b >= 0;
       b = din_next_sample(sched, B, static_b, gridDim.x * WARPS, lane)) {
    // ---------------- per-sample preparation
    __syncwarp();
    for (int i = lane; i < T * H; i += 32) skeys[i] = __ldg(keys + (size_t)b * T * H + i);
    for (int i = lane; i < H; i += 32) { sq[i] = __ldg(query + (size_t)b * H + i); sgo[i] = __ldg(g_out + (size_t)b * H + i); }
    __syncwarp();
    float weff[HP][2], kd[HP][2], qpart[2], dsum[2] = {0.f, 0.f};
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int c = lane + 32 * u;
      float acc = sm[L.b1 + c];
#pragma unroll
      for (int h = 0; h < HP; ++h) {
        kd[h][u] = 0.f;
        if (h < H) {
          const float qh = sq[h];
          acc += qh * sm[L.wq + h * DIN_H1 + c];
          weff[h][u] = sm[L.wk + h * DIN_H1 + c] + qh * sm[L.wd + h * DIN_H1 + c];
        } else {
          weff[h][u] = 0.f;
        }
        swt[c * (HP + 1) + h] = weff[h][u];
      }
      qpart[u] = acc;
    }
    long long len64 = __ldg(keys_length + b);
    const int len = (int)(len64 < 0 ? 0 : (len64 > T ? T : len64));
    // ---------------- attention weights: saved by the forward, or recomputed
    if (att_w != nullptr) {
      for (int t = lane; t < T; t += 32) sc[t] = __ldg(att_w + (size_t)b * T + t);
      __syncwarp();
    } else {
      for (int t = 0; t < len; ++t) {
        float h1a, h1b, h2, score;
        mlp_fwd(skeys + t * H, weff, qpart, h1a, h1b, h2, score);
        if (lane == 0) sc[t] = score;
        __syncwarp();
      }
      din_weights(sc, T, len, H, is_softmax, lane);
    }
    // dw[t] = go . k[t];  dkeys[t,:] = w[t]*go;  ds from the mask / softmax backward
    float dot = 0.f;
    for (int t = lane; t < T; t += 32) {
      float dwv = 0.f;
      for (int h = 0; h < H; ++h) dwv += sgo[h] * skeys[t * H + h];
      sds[t] = dwv;
      dot += sc[t] * dwv;
    }
    dot = warp_sum(dot);
    const float scale = sqrtf((float)H);
    for (int t = lane; t < T; t += 32) {
      const float dwv = sds[t];
      sds[t] = t < len ? (is_softmax ? sc[t] * (dwv - dot) / scale : dwv) : 0.f;
    }
    // d_keys = w[t]*go (every position, padded ones included) + Weff.dpre1[t] (t < len, added below by the lanes that own (t,h))
    for (int i = lane; i < T * H; i += 32) {
      const int t = i / H;
      if (t >= len) d_keys[(size_t)b * T * H + i] = sc[t] * sgo[i - t * H];
    }
    __syncwarp();
    // ---------------- positions, DIN_BT at a time: every shared-memory round trip (h1 broadcast, W2 column/row chunks, Weff^T)
    // and every warp sync serves DIN_BT positions; accumulators stay in registers
    for (int t0 = 0; t0 < len; t0 += DIN_BT) {
      const int n = min(DIN_BT, len - t0);
      float h1a[DIN_BT], h1b[DIN_BT], dp2[DIN_BT];
#pragma unroll
      for (int tt = 0; tt < DIN_BT; ++tt) {
        float p0 = qpart[0], p1 = qpart[1];
        const float* k = skeys + (t0 + (tt < n ? tt : 0)) * H;
#pragma unroll
        for (int h = 0; h < HP; ++h) {
          if (h < H) {
            const float kv = k[h];
            p0 += kv * weff[h][0];
            p1 += kv * weff[h][1];
          }
        }
        h1a[tt] = tt < n ? fmaxf(p0, 0.f) : 0.f;
        h1b[tt] = tt < n ? fmaxf(p1, 0.f) : 0.f;
        sh1[tt * DIN_H1 + lane] = h1a[tt];
        sh1[tt * DIN_H1 + lane + 32] = h1b[tt];
      }
      __syncwarp();
      {
        float acc[DIN_BT];
#pragma unroll
        for (int tt = 0; tt < DIN_BT; ++tt) acc[tt] = b2v;
#pragma unroll
        for (int c4 = 0; c4 < DIN_H1 / 4; ++c4) {
          const float w0 = W2s[(4 * c4 + 0) * DIN_H2 + lane], w1v = W2s[(4 * c4 + 1) * DIN_H2 + lane],
                      w2v = W2s[(4 * c4 + 2) * DIN_H2 + lane], w3c = W2s[(4 * c4 + 3) * DIN_H2 + lane];
#pragma unroll
          for (int tt = 0; tt < DIN_BT; ++tt) {
            const float4 hv = reinterpret_cast<const float4*>(sh1 + tt * DIN_H1)[c4];
            acc[tt] += hv.x * w0; acc[tt] += hv.y * w1v; acc[tt] += hv.z * w2v; acc[tt] += hv.w * w3c;
          }
        }
#pragma unroll
        for (int tt = 0; tt < DIN_BT; ++tt) {
          const float h2 = fmaxf(acc[tt], 0.f);
          const float dsv = tt < n ? sds[t0 + tt] : 0.f;
          dp2[tt] = h2 > 0.f ? dsv * w3v : 0.f;
          sdp2[tt * DIN_H2 + lane] = dp2[tt];
          acc_w3 += h2 * dsv;
          acc_b2 += dp2[tt];
          acc_b3 += dsv;
        }
      }
      // dW2[:, lane] += sum_tt h1[tt][:] * dpre2[tt][lane]
#pragma unroll
      for (int c4 = 0; c4 < DIN_H1 / 4; ++c4) {
#pragma unroll
        for (int tt = 0; tt < DIN_BT; ++tt) {
          const float4 hv = reinterpret_cast<const float4*>(sh1 + tt * DIN_H1)[c4];
          acc_w2[4 * c4 + 0] += hv.x * dp2[tt]; acc_w2[4 * c4 + 1] += hv.y * dp2[tt];
          acc_w2[4 * c4 + 2] += hv.z * dp2[tt]; acc_w2[4 * c4 + 3] += hv.w * dp2[tt];
        }
      }
      __syncwarp();
      // dh1[tt][c] = sum_c2 dpre2[tt][c2] * W2[c][c2] for c = lane, lane+32 (rotated 16-byte chunks: conflict-free)
      float d0[DIN_BT], d1[DIN_BT];
      {
        float a0[DIN_BT], a1[DIN_BT];
#pragma unroll
        for (int tt = 0; tt < DIN_BT; ++tt) { a0[tt] = 0.f; a1[tt] = 0.f; }
        const float4* r0 = reinterpret_cast<const float4*>(W2s + lane * DIN_H2);
        const float4* r1 = reinterpret_cast<const float4*>(W2s + (lane + 32) * DIN_H2);
#pragma unroll
        for (int c4 = 0; c4 < DIN_H2 / 4; ++c4) {
          const int ch = (c4 + lane) & (DIN_H2 / 4 - 1);
          const float4 x0 = r0[ch], x1 = r1[ch];
#pragma unroll
          for (int tt = 0; tt < DIN_BT; ++tt) {
            const float4 dd = reinterpret_cast<const float4*>(sdp2 + tt * DIN_H2)[ch];
            a0[tt] += dd.x * x0.x + dd.y * x0.y + dd.z * x0.z + dd.w * x0.w;
            a1[tt] += dd.x * x1.x + dd.y * x1.y + dd.z * x1.z + dd.w * x1.w;
          }
        }
#pragma unroll
        for (int tt = 0; tt < DIN_BT; ++tt) {
          d0[tt] = h1a[tt] > 0.f ? a0[tt] : 0.f;
          d1[tt] = h1b[tt] > 0.f ? a1[tt] : 0.f;
          dsum[0] += d0[tt]; dsum[1] += d1[tt];
          sdp1[tt * DIN_H1 + lane] = d0[tt]; sdp1[tt * DIN_H1 + lane + 32] = d1[tt];
        }
      }
#pragma unroll
      for (int tt = 0; tt < DIN_BT; ++tt) {
        const float* k = skeys + (t0 + (tt < n ? tt : 0)) * H;       // d0 = d1 = 0 beyond n
#pragma unroll
        for (int h = 0; h < HP; ++h) {
          if (h < H) {
            const float kv = k[h];
            kd[h][0] += kv * d0[tt];
            kd[h][1] += kv * d1[tt];
          }
        }
      }
      __syncwarp();
      // dk[t][h] += sum_c Weff[h][c] * dpre1[t][c] : lane = (group, h); every group covers 64/ngroups columns
      {
        constexpr int NG = 32 / HP;                 // groups of HP lanes
        constexpr int CPG = DIN_H1 / NG;            // columns per group
        const int hh = lane % HP, grp = lane / HP;
        float part[DIN_BT];
#pragma unroll
        for (int tt = 0; tt < DIN_BT; ++tt) part[tt] = 0.f;
#pragma unroll 8
        for (int cc = 0; cc < CPG; ++cc) {
          const int c = grp * CPG + cc;
          const float wv = swt[c * (HP + 1) + hh];
#pragma unroll
          for (int tt = 0; tt < DIN_BT; ++tt) part[tt] += sdp1[tt * DIN_H1 + c] * wv;
        }
#pragma unroll
        for (int tt = 0; tt < DIN_BT; ++tt) {
#pragma unroll
          for (int o = HP; o < 32; o <<= 1) part[tt] += __shfl_xor_sync(0xffffffffu, part[tt], o);
          if (grp == 0 && hh < H && tt < n)
            d_keys[((size_t)b * T + t0 + tt) * H + hh] = sc[t0 + tt] * sgo[hh] + part[tt];
        }
      }
      __syncwarp();
    }
    // ---------------- sample epilogue: d_query, d_keys, flush the layer-1 weight-gradient pieces
    const int c0 = lane, c1 = lane + 32;
#pragma unroll
    for (int h = 0; h < HP; ++h) {
      if (h < H) {
        float v = sm[L.wq + h * DIN_H1 + c0] * dsum[0] + sm[L.wq + h * DIN_H1 + c1] * dsum[1] +
                  sm[L.wd + h * DIN_H1 + c0] * kd[h][0] + sm[L.wd + h * DIN_H1 + c1] * kd[h][1];
        v = warp_sum(v);
        if (lane == 0) d_query[(size_t)b * H + h] = v;
        const float qh = sq[h];
        float* pa = pacc + h * DIN_H1;
        float* pb = pa + H * DIN_H1;
        float* pd = pb + H * DIN_H1;
        pa[c0] += qh * dsum[0]; pa[c1] += qh * dsum[1];
        pb[c0] += kd[h][0];     pb[c1] += kd[h][1];
        pd[c0] += qh * kd[h][0]; pd[c1] += qh * kd[h][1];
      }
    }
    pacc[3 * H * DIN_H1 + c0] += dsum[0];
    pacc[3 * H * DIN_H1 + c1] += dsum[1];
  }
  // ---------------- merge: warp registers -> CTA shared accumulators -> global
#pragma unroll
  for (int c = 0; c < DIN_H1; ++c) atomicAdd(sm + L.aw2 + c * DIN_H2 + lane, acc_w2[c]);
  atomicAdd(sm + L.ab2 + lane, acc_b2);
  atomicAdd(sm + L.aw3 + lane, acc_w3);
  if (lane == 0) atomicAdd(sm + L.aw3 + DIN_H2, acc_b3);
  __syncthreads();
  float* dW1 = d_params;
  float* dB1 = dW1 + H4 * DIN_H1;
  float* dW2 = dB1 + DIN_H1;
  float* dB2 = dW2 + DIN_H1 * DIN_H2;
  float* dW3 = dB2 + DIN_H2;
  float* dB3 = dW3 + DIN_H2;
  const float* pw0 = sm + L.per_warp + L.o_acc;           // warp w's private sums start at pw0 + w * warp_stride
  for (int i = tid; i < H * DIN_H1; i += blockDim.x) {
    float a = 0.f, bb = 0.f, d = 0.f;
#pragma unroll
    for (int wv = 0; wv < WARPS; ++wv) {
      const float* pw = pw0 + (size_t)wv * L.warp_stride;
      a += pw[i]; bb += pw[H * DIN_H1 + i]; d += pw[2 * H * DIN_H1 + i];
    }
    atomicAdd(dW1 + i, a);
    atomicAdd(dW1 + H * DIN_H1 + i, bb);
    atomicAdd(dW1 + 2 * H * DIN_H1 + i, a - bb);
    atomicAdd(dW1 + 3 * H * DIN_H1 + i, d);
  }
  for (int i = tid; i < DIN_H1; i += blockDim.x) {
    float v = 0.f;
#pragma unroll
    for (int wv = 0; wv < WARPS; ++wv) v += pw0[(size_t)wv * L.warp_stride + 3 * H * DIN_H1 + i];
    atomicAdd(dB1 + i, v);
  }
  for (int i = tid; i < DIN_H1 * DIN_H2; i += blockDim.x) atomicAdd(dW2 + i, sm[L.aw2 + i]);
  for (int i = tid; i < DIN_H2; i += blockDim.x) { atomicAdd(dB2 + i, sm[L.ab2 + i]); atomicAdd(dW3 + i, sm[L.aw3 + i]); }
  if (tid == 0) atomicAdd(dB3, sm[L.aw3 + DIN_H2]);
}

}  // namespace ctr

using namespace ctr;

static int check_din(const char* fn, int64_t B, int64_t T, int64_t H) {
  CTR_REQUIRE(B >= 0 && T >= 0 && H >= 1, "%s: bad sizes B=%lld T=%lld H=%lld", fn, (long long)B, (long long)T,
              (long long)H);
  CTR_UNSUPPORTED(H > 32, "%s: H=%lld > 32 unsupported", fn, (long long)H);
  return CTR_OK;
}

static int din_fwd_launch(const float* query, const float* keys, const int64_t* len, const float* w1, const float* b1,
                          const float* w2, const float* b2, const float* w3, const float* b3, int64_t B, int64_t T,
                          int64_t H, int is_softmax, float* out, float* att_w, int* sched, cudaStream_t st) {
  constexpr int WARPS = 4;
  const DinSmem L = din_layout((int)H, (int)T, WARPS, false);
  const size_t smem = sizeof(float) * (size_t)L.total;
  CTR_UNSUPPORTED(smem > 220 * 1024, "ctr_din_attention_fwd: T=%lld H=%lld needs %zu B of shared memory", (long long)T,
                  (long long)H, smem);
  return with_const<4, 8, 16, 32>(H <= 4 ? 4 : H <= 8 ? 8 : H <= 16 ? 16 : 32, [&](auto HPV) {
    return launch_resident("ctr_din_attention_fwd", din_attention_fwd_kernel<HPV, WARPS>, (B + WARPS - 1) / WARPS, WARPS * 32, smem, st,
                           query, keys, reinterpret_cast<const long long*>(len), w1, b1, w2, b2, w3, b3, (int)B, (int)T, (int)H,
                           is_softmax, out, att_w, sched);
  });
}

extern "C" int ctr_din_attention_fwd(const float* query, const float* keys, const int64_t* keys_length, const float* w1,
                                     const float* b1, const float* w2, const float* b2, const float* w3,
                                     const float* b3, int64_t B, int64_t T, int64_t H, int is_softmax, float* out,
                                     float* att_w, int32_t* sched_scratch, void* stream) {
  int rc = check_din("ctr_din_attention_fwd", B, T, H);
  if (rc) return rc;
  CTR_REQUIRE(query && keys_length && w1 && b1 && w2 && b2 && w3 && b3 && out && (keys || T == 0),
              "ctr_din_attention_fwd: null argument");
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  if (T == 0) {                                           // empty history: the weighted sum over no keys is 0
    CTR_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * B * H, st));
    return CTR_OK;
  }
  if (sched_scratch != nullptr) {
    CTR_UNSUPPORTED(T > 8192, "ctr_din_attention_fwd: T=%lld too long for the schedule pass", (long long)T);
    rc = launch("ctr_din_attention_fwd(schedule)", din_schedule_kernel, 1, 1024, sizeof(int) * (T + 2), st,
                reinterpret_cast<const long long*>(keys_length), (int)B, (int)T, sched_scratch);
    if (rc) return rc;
  }
  return din_fwd_launch(query, keys, keys_length, w1, b1, w2, b2, w3, b3, B, T, H, is_softmax, out, att_w, sched_scratch, st);
}

extern "C" int ctr_din_attention_bwd(const float* query, const float* keys, const int64_t* keys_length, const float* w1,
                                     const float* b1, const float* w2, const float* b2, const float* w3,
                                     const float* b3, const float* g_out, const float* att_w, int64_t B, int64_t T,
                                     int64_t H, int is_softmax, float* d_query, float* d_keys, float* d_params,
                                     int32_t* sched_scratch, void* stream) {
  int rc = check_din("ctr_din_attention_bwd", B, T, H);
  if (rc) return rc;
  CTR_REQUIRE(query && keys_length && w1 && b1 && w2 && b2 && w3 && b3 && g_out && d_query && d_params &&
                  ((keys && d_keys) || T == 0), "ctr_din_attention_bwd: null argument");
  cudaStream_t st = as_stream(stream);
  const int64_t nparams = 4 * H * DIN_H1 + DIN_H1 + DIN_H1 * DIN_H2 + DIN_H2 + DIN_H2 + 1;
  CTR_CUDA(cudaMemsetAsync(d_params, 0, sizeof(float) * nparams, st));
  if (B == 0) return CTR_OK;
  if (T == 0) {
    CTR_CUDA(cudaMemsetAsync(d_query, 0, sizeof(float) * B * H, st));
    return CTR_OK;
  }
  if (sched_scratch != nullptr) {
    CTR_UNSUPPORTED(T > 8192, "ctr_din_attention_bwd: T=%lld too long for the schedule pass", (long long)T);
    rc = launch("ctr_din_attention_bwd(schedule)", din_schedule_kernel, 1, 1024, sizeof(int) * (T + 2), st,
                reinterpret_cast<const long long*>(keys_length), (int)B, (int)T, sched_scratch);
    if (rc) return rc;
  }
  const int HPv = H <= 4 ? 4 : H <= 8 ? 8 : H <= 16 ? 16 : 32;
  // 8 warps per CTA unless their staging areas do not fit the shared memory (long sequences of wide keys): then 4
  const bool w8 = sizeof(float) * (size_t)din_bwd_layout((int)H, HPv, (int)T, 8).total <= 220 * 1024;
  const int warps = w8 ? 8 : 4;
  const DinBwdSmem L = din_bwd_layout((int)H, HPv, (int)T, warps);
  const size_t smem = sizeof(float) * (size_t)L.total;
  CTR_UNSUPPORTED(smem > 220 * 1024, "ctr_din_attention_bwd: T=%lld H=%lld needs %zu B of shared memory", (long long)T,
                  (long long)H, smem);
  return with_const<4, 8, 16, 32>(HPv, [&](auto HPV) {
    return with_const<4, 8>(warps, [&](auto WARPS) {
      return launch_resident("ctr_din_attention_bwd", din_attention_bwd_kernel<HPV, WARPS>, (B + WARPS - 1) / WARPS, WARPS * 32, smem,
                             st, query, keys, reinterpret_cast<const long long*>(keys_length), w1, b1, w2, b2, w3, b3, g_out, att_w,
                             (int)B, (int)T, (int)H, is_softmax, d_query, d_keys, d_params, sched_scratch);
    });
  });
}

// Row CROSS (SURVEY.md section 8a): the DCN cross-layer stack, all L layers in one launch.
//
// Reference: cross_layer(x0, xl, index) -- DCN/cross_layer.py:21-24 -- stacked by the loop at
// DCN/dcn.py:157-160:   x_{l+1} = x0 * (x_l . w_l) + b_l + x_l   (w_l, b_l are (d,1) variables).
//
// H100 mapping (HBM/L2-bound, 20*d bytes per sample fwd+bwd; no tensor cores):
//   forward : one warp per sample, x0 and x_l live in registers (d/32 values per lane), w/b of all layers
//             staged once per CTA in shared memory, the (B,d)x(d,1) product is a warp-shuffle dot.
//   backward: phase 1 (warp per sample) re-runs the forward recurrence to get s_l = x_l.w_l, then walks
//             the layers backwards keeping g in registers (t_l = g.x0, dx0 += g*s_l, g += t_l*w_l);
//             phase 2 (thread per column) forms the batch reductions dw_l = sum_b x_l*t_l and
//             db_l = sum_b g_{l+1} from the tile staged in shared memory, using
//                 x_l     = xs + x0 * sum_{k<l} s_k + sum_{k<l} b_k        (xs = start vector)
//                 g_{l+1} = g_out + sum_{k>l} t_k * w_k
//             so no per-layer activations are ever written to HBM; per-CTA partials are merged with
//             fp32 atomics.
#include <type_traits>

#include "ctr_common.cuh"

namespace ctr {

constexpr int CROSS_WARPS = 8;          // samples per CTA iteration
constexpr int CROSS_LMAX = 8;           // layers supported by the fused backward

// N = ceil(d / (32*VEC)) element groups per lane; element index of (k, lane, v) = (k*32 + lane)*VEC + v
template <int VEC, int N>
struct LaneVec {
  float v[N * VEC];
  __device__ __forceinline__ void load(const float* __restrict__ p, int d, int lane) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const int i = (k * 32 + lane) * VEC;
      if constexpr (VEC == 4) {
        float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < d) t = __ldg(reinterpret_cast<const float4*>(p + i));
        v[k * 4 + 0] = t.x; v[k * 4 + 1] = t.y; v[k * 4 + 2] = t.z; v[k * 4 + 3] = t.w;
      } else {
        v[k] = i < d ? __ldg(p + i) : 0.f;
      }
    }
  }
  // plain (generic-address) store: used for both global outputs and the shared-memory tile
  __device__ __forceinline__ void store(float* __restrict__ p, int d, int lane) const {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const int i = (k * 32 + lane) * VEC;
      if (i < d) {
        if constexpr (VEC == 4)
          *reinterpret_cast<float4*>(p + i) = make_float4(v[k * 4 + 0], v[k * 4 + 1], v[k * 4 + 2], v[k * 4 + 3]);
        else
          p[i] = v[k];
      }
    }
  }
};

template <int VEC, int N>
__device__ __forceinline__ void lane_load_smem(float (&r)[N * VEC], const float* s, int d, int lane) {
#pragma unroll
  for (int k = 0; k < N; ++k) {
    const int i = (k * 32 + lane) * VEC;
    if constexpr (VEC == 4) {
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
      if (i < d) t = *reinterpret_cast<const float4*>(s + i);
      r[k * 4 + 0] = t.x; r[k * 4 + 1] = t.y; r[k * 4 + 2] = t.z; r[k * 4 + 3] = t.w;
    } else {
      r[k] = i < d ? s[i] : 0.f;
    }
  }
}

template <int VEC, int N>
__global__ void __launch_bounds__(CROSS_WARPS * 32)
cross_fwd_kernel(const float* __restrict__ x0, const float* __restrict__ xl_in, const float* __restrict__ w,
                 const float* __restrict__ b, int B, int d, int L, float* __restrict__ out) {
  extern __shared__ __align__(16) float smem[];
  float* sw = smem;                  // (L, d)
  float* sb = smem + (size_t)L * d;  // (L, d)
  for (int i = threadIdx.x; i < L * d; i += blockDim.x) { sw[i] = __ldg(w + i); sb[i] = __ldg(b + i); }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int s = warp0; s < B; s += nwarps) {
    LaneVec<VEC, N> a0, x;
    a0.load(x0 + (size_t)s * d, d, lane);
    if (xl_in) x.load(xl_in + (size_t)s * d, d, lane);
    else {
#pragma unroll
      for (int k = 0; k < N * VEC; ++k) x.v[k] = a0.v[k];
    }
    for (int l = 0; l < L; ++l) {
      float wv[N * VEC], bv[N * VEC];
      lane_load_smem<VEC, N>(wv, sw + (size_t)l * d, d, lane);
      lane_load_smem<VEC, N>(bv, sb + (size_t)l * d, d, lane);
      float dot = 0.f;
#pragma unroll
      for (int k = 0; k < N * VEC; ++k) dot += x.v[k] * wv[k];
      dot = warp_sum(dot);                                            // xl_wl  (B,1)
#pragma unroll
      for (int k = 0; k < N * VEC; ++k) x.v[k] = (a0.v[k] * dot + bv[k]) + x.v[k];   // (x0*xl_wl + bl^T) + xl
    }
    x.store(out + (size_t)s * d, d, lane);
  }
}

__device__ __forceinline__ void cp_async16(unsigned smem_dst, const float* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gsrc) : "memory");
}

// CPT = ceil(d / blockDim) columns per thread in phase 2.
// PF: the (x0, xs, g) tiles of the NEXT iteration are fetched with cp.async into a second shared-memory buffer while
// this iteration computes (the kernel is otherwise bound by exposed global-load latency: 8 warps/SM, one sample each).
template <int VEC, int N, int CPT, bool PF, int LM>
__global__ void __launch_bounds__(CROSS_WARPS * 32)
cross_bwd_kernel(const float* __restrict__ x0, const float* __restrict__ xl_in, const float* __restrict__ w,
                 const float* __restrict__ b, const float* __restrict__ g_out, int B, int d, int L,
                 float* __restrict__ dx0, float* __restrict__ dxl_in, float* __restrict__ dw,
                 float* __restrict__ db) {
  extern __shared__ __align__(16) float smem[];
  float* sw = smem;                                  // (L, d)  weights
  float* sb = sw + (size_t)L * d;                    // (L, d)  biases
  float* scb = sb + (size_t)L * d;                   // (L, d)  prefix biases  cb_l = sum_{k<l} b_k
  const int narr = xl_in ? 3 : 2;                    // tiles per buffer: x0, [xs], g
  const size_t buf_floats = (size_t)narr * CROSS_WARPS * d;
  float* tiles0 = scb + (size_t)L * d;               // buffer 0 (and buffer 1 right behind it when PF)
  float* scs = tiles0 + (PF ? 2 : 1) * buf_floats;   // (W, LMAX)  cs_l = sum_{k<l} s_k
  float* st = scs + CROSS_WARPS * LM;        // (W, LMAX)  t_l
  __shared__ int s_valid[CROSS_WARPS];

  for (int i = threadIdx.x; i < L * d; i += blockDim.x) { sw[i] = __ldg(w + i); sb[i] = __ldg(b + i); }
  __syncthreads();
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    float acc = 0.f;
    for (int l = 0; l < L; ++l) { scb[(size_t)l * d + i] = acc; acc += sb[(size_t)l * d + i]; }
  }
  const int lane = threadIdx.x & 31;
  const int wid = threadIdx.x >> 5;
  float acc_dw[LM][CPT], acc_db[LM][CPT];
#pragma unroll
  for (int l = 0; l < LM; ++l)
#pragma unroll
    for (int c = 0; c < CPT; ++c) { acc_dw[l][c] = 0.f; acc_db[l][c] = 0.f; }
  __syncthreads();

  const int ntiles = (B + CROSS_WARPS - 1) / CROSS_WARPS;
  const unsigned tiles_u32 = (unsigned)__cvta_generic_to_shared(tiles0);
  auto issue_tile = [&](int tile, int buf) {          // cp.async the tile's contiguous 8*d floats of each array
    const unsigned base = tiles_u32 + (unsigned)(buf * buf_floats * sizeof(float));
    const long long first = (long long)tile * CROSS_WARPS;
    const int nfl = (int)min((long long)CROSS_WARPS, (long long)B - first) * d;
    const unsigned arr_bytes = (unsigned)(CROSS_WARPS * d * sizeof(float));
    for (int i = threadIdx.x * 4; i < nfl; i += blockDim.x * 4) {
      cp_async16(base + 4u * i, x0 + first * d + i);
      if (xl_in) cp_async16(base + arr_bytes + 4u * i, xl_in + first * d + i);
      cp_async16(base + (narr - 1) * arr_bytes + 4u * i, g_out + first * d + i);
    }
  };
  int buf = 0;
  if (PF) {
    if ((int)blockIdx.x < ntiles) issue_tile(blockIdx.x, 0);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int s = tile * CROSS_WARPS + wid;
    float* tx0 = tiles0 + (size_t)(PF ? buf : 0) * buf_floats;
    float* txs = xl_in ? tx0 + (size_t)CROSS_WARPS * d : tx0;
    float* tg = tx0 + (size_t)(narr - 1) * CROSS_WARPS * d;
    if (PF) {
      const int next = tile + gridDim.x;
      if (next < ntiles) issue_tile(next, buf ^ 1);
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 1;" ::: "memory");     // this iteration's tile has landed
      __syncthreads();
    }
    // ---------------- phase 1: warp per sample ----------------
    if (lane == 0) s_valid[wid] = s < B;
    if (s < B) {
      LaneVec<VEC, N> a0, x, g;
      if (PF) {
        lane_load_smem<VEC, N>(a0.v, tx0 + (size_t)wid * d, d, lane);
        lane_load_smem<VEC, N>(x.v, txs + (size_t)wid * d, d, lane);
        lane_load_smem<VEC, N>(g.v, tg + (size_t)wid * d, d, lane);
      } else {
        a0.load(x0 + (size_t)s * d, d, lane);
        if (xl_in) x.load(xl_in + (size_t)s * d, d, lane);
        else {
#pragma unroll
          for (int k = 0; k < N * VEC; ++k) x.v[k] = a0.v[k];
        }
        g.load(g_out + (size_t)s * d, d, lane);
        a0.store(tx0 + (size_t)wid * d, d, lane);
        if (xl_in) x.store(txs + (size_t)wid * d, d, lane);
        g.store(tg + (size_t)wid * d, d, lane);
      }
      // forward recurrence -> s_l (kept in registers of every lane), prefix sums to smem
      float sl[LM];
      float cs = 0.f;
#pragma unroll
      for (int l = 0; l < LM; ++l) {
        sl[l] = 0.f;
        if (l < L) {
          float wv[N * VEC], bv[N * VEC];
          lane_load_smem<VEC, N>(wv, sw + (size_t)l * d, d, lane);
          lane_load_smem<VEC, N>(bv, sb + (size_t)l * d, d, lane);
          float dot = 0.f;
#pragma unroll
          for (int k = 0; k < N * VEC; ++k) dot += x.v[k] * wv[k];
          dot = warp_sum(dot);
          sl[l] = dot;
          if (lane == 0) scs[wid * LM + l] = cs;
          cs += dot;
#pragma unroll
          for (int k = 0; k < N * VEC; ++k) x.v[k] = (a0.v[k] * dot + bv[k]) + x.v[k];
        }
      }
      // backward walk; x now reused as the dx0 accumulator
#pragma unroll
      for (int k = 0; k < N * VEC; ++k) x.v[k] = 0.f;
#pragma unroll
      for (int l = LM - 1; l >= 0; --l) {
        if (l < L) {
          float wv[N * VEC];
          lane_load_smem<VEC, N>(wv, sw + (size_t)l * d, d, lane);
          float t = 0.f;
#pragma unroll
          for (int k = 0; k < N * VEC; ++k) t += g.v[k] * a0.v[k];
          t = warp_sum(t);
          if (lane == 0) st[wid * LM + l] = t;
#pragma unroll
          for (int k = 0; k < N * VEC; ++k) {
            x.v[k] += g.v[k] * sl[l];
            g.v[k] += t * wv[k];
          }
        }
      }
      if (xl_in) {
        g.store(dxl_in + (size_t)s * d, d, lane);
      } else {
#pragma unroll
        for (int k = 0; k < N * VEC; ++k) x.v[k] += g.v[k];
      }
      x.store(dx0 + (size_t)s * d, d, lane);
    }
    __syncthreads();
    // ---------------- phase 2: thread per column ----------------
#pragma unroll
    for (int c = 0; c < CPT; ++c) {
      const int i = c * (CROSS_WARPS * 32) + threadIdx.x;
      if (i < d) {
        for (int q = 0; q < CROSS_WARPS; ++q) {
          if (!s_valid[q]) continue;
          const float vx0 = tx0[(size_t)q * d + i], vxs = txs[(size_t)q * d + i];
          float gl = tg[(size_t)q * d + i];
#pragma unroll
          for (int l = LM - 1; l >= 0; --l) {
            if (l < L) {
              const float t = st[q * LM + l];
              const float xl = (vx0 * scs[q * LM + l] + scb[(size_t)l * d + i]) + vxs;
              acc_dw[l][c] += xl * t;
              acc_db[l][c] += gl;
              gl += t * sw[(size_t)l * d + i];
            }
          }
        }
      }
    }
    __syncthreads();
    buf ^= 1;
  }
#pragma unroll
  for (int c = 0; c < CPT; ++c) {
    const int i = c * (CROSS_WARPS * 32) + threadIdx.x;
    if (i < d) {
#pragma unroll
      for (int l = 0; l < LM; ++l) {
        if (l < L) {
          atomicAdd(dw + (size_t)l * d + i, acc_dw[l][c]);
          atomicAdd(db + (size_t)l * d + i, acc_db[l][c]);
        }
      }
    }
  }
}

// Backward, register form (the common case: xl_in == x0 chain, L <= 4, d % 4 == 0): NO per-iteration block phases.
// With xs == x0 the batch reductions factor through per-sample scalars:
//     dw_l[i] = sum_q x0[q,i] * a_l(q)  +  cb_l[i] * T_l          a_l = (1 + sum_{k<l} s_k) * t_l ,  T_l = sum_q t_l(q)
//     db_l[i] = sum_q g_out[q,i]        +  sum_{k>l} w_k[i] * T_k
// so the warp that owns a sample adds x0*a_l and g_out into lane-owned register accumulators (columns of the lane) while the
// values are still in its registers; nothing is staged in shared memory, there is no thread-per-column phase and no
// __syncthreads in the loop (the first form spent ~60 % of its issue slots in that phase and two block syncs per 8 samples).
// Second step (ncu: six DEPENDENT warp reductions per sample kept 8 warps/SM latency-bound at 36 % of HBM): with x_l affine in
// x0 the whole layer chain becomes scalar recurrences over L + 1 independent dot products (see the loop body).
// The next sample's x0 / g_out are fetched one iteration ahead.  Per CTA: one shared-memory reduction, then the cb / w terms
// and one fp32 atomic per element.
template <int N, int LM, int RW>
__global__ void __launch_bounds__(RW * 32)
cross_bwd_reg_kernel(const float* __restrict__ x0, const float* __restrict__ w, const float* __restrict__ b,
                     const float* __restrict__ g_out, int B, int d, int L, float* __restrict__ dx0,
                     float* __restrict__ dw, float* __restrict__ db) {
  constexpr int NV = N * 4;
  extern __shared__ __align__(16) float smem[];
  float* sw = smem;                                  // (L, d)  weights
  float* sb = sw + (size_t)L * d;                    // (L, d)  biases
  float* part = sb + (size_t)L * d;                  // (RW, (L+1)*d)  per-warp partial sums: sum_q x0*a_l (l < L) and sum_q g_out
  float* partT = part + (size_t)RW * (L + 1) * d;    // (RW, LM)       per-warp T_l
  for (int i = threadIdx.x; i < L * d; i += blockDim.x) { sw[i] = __ldg(w + i); sb[i] = __ldg(b + i); }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  float acc_a[LM][NV], acc_g[NV], T[LM];
#pragma unroll
  for (int l = 0; l < LM; ++l) {
    T[l] = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) acc_a[l][k] = 0.f;
  }
#pragma unroll
  for (int k = 0; k < NV; ++k) acc_g[k] = 0.f;
  // v_l = cb_l . w_l (sample independent): the bias part of s_l = x_l . w_l with x_l = x0*(1 + cs_l) + cb_l
  float vl[LM];
  {
    float cbv[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) cbv[k] = 0.f;
#pragma unroll
    for (int l = 0; l < LM; ++l) {
      vl[l] = 0.f;
      if (l < L) {
        float wv[NV], bv[NV];
        lane_load_smem<4, N>(wv, sw + (size_t)l * d, d, lane);
        lane_load_smem<4, N>(bv, sb + (size_t)l * d, d, lane);
        float dot = 0.f;
#pragma unroll
        for (int k = 0; k < NV; ++k) { dot += cbv[k] * wv[k]; cbv[k] += bv[k]; }
        vl[l] = warp_sum(dot);
      }
    }
  }
  LaneVec<4, N> na0, ng;
  if (warp0 < B) { na0.load(x0 + (size_t)warp0 * d, d, lane); ng.load(g_out + (size_t)warp0 * d, d, lane); }
  for (int s = warp0; s < B; s += nwarps) {
    LaneVec<4, N> a0 = na0, g = ng;
    if (s + nwarps < B) { na0.load(x0 + (size_t)(s + nwarps) * d, d, lane); ng.load(g_out + (size_t)(s + nwarps) * d, d, lane); }
    // The only reductions a sample needs are L + 1 INDEPENDENT dot products -- u_l = x0 . w_l and c0 = g_out . x0 -- done as one
    // batched butterfly; everything sequential in the layer chain collapses to scalar recurrences:
    //   s_l = (1 + cs_l) u_l + v_l ,  cs_{l+1} = cs_l + s_l          (forward:  x_l = x0 (1 + cs_l) + cb_l)
    //   t_l = c0 + sum_{k>l} t_k u_k                                 (backward: g_{l+1} = g_out + sum_{k>l} t_k w_k)
    //   dx0 = g_out (1 + cs_L) + sum_k a_k w_k ,  a_k = (1 + cs_k) t_k     (a_k is also the dw scalar)
    float red[LM + 1];
#pragma unroll
    for (int l = 0; l <= LM; ++l) red[l] = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) { red[LM] += g.v[k] * a0.v[k]; acc_g[k] += g.v[k]; }
#pragma unroll
    for (int l = 0; l < LM; ++l) {
      if (l < L) {
        float wv[NV];
        lane_load_smem<4, N>(wv, sw + (size_t)l * d, d, lane);
#pragma unroll
        for (int k = 0; k < NV; ++k) red[l] += a0.v[k] * wv[k];
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int l = 0; l <= LM; ++l) red[l] += __shfl_xor_sync(0xffffffffu, red[l], o);
    }
    float cs[LM + 1], tl[LM], al[LM];
    cs[0] = 0.f;
#pragma unroll
    for (int l = 0; l < LM; ++l) cs[l + 1] = l < L ? cs[l] + ((1.f + cs[l]) * red[l] + vl[l]) : cs[l];
    float run = 0.f;                                   // sum_{k>l} t_k u_k
#pragma unroll
    for (int l = LM - 1; l >= 0; --l) {
      tl[l] = 0.f; al[l] = 0.f;
      if (l < L) {
        tl[l] = red[LM] + run;
        run += tl[l] * red[l];
        al[l] = (1.f + cs[l]) * tl[l];
        T[l] += tl[l];
      }
    }
    const float gscale = 1.f + cs[LM];                 // cs[LM] == cs_L for every l >= L
    LaneVec<4, N> x;
#pragma unroll
    for (int k = 0; k < NV; ++k) x.v[k] = g.v[k] * gscale;
#pragma unroll
    for (int l = 0; l < LM; ++l) {
      if (l < L) {
        float wv[NV];
        lane_load_smem<4, N>(wv, sw + (size_t)l * d, d, lane);
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          x.v[k] += al[l] * wv[k];
          acc_a[l][k] += a0.v[k] * al[l];
        }
      }
    }
    x.store(dx0 + (size_t)s * d, d, lane);
  }
  // ---- CTA reduction of the lane-owned accumulators: every warp parks its partial sums in its own slice of shared memory
  // (128-bit stores, no ordering between warps), one barrier, then thread-per-column sums over the RW slices.  (The first form
  // let the warps take turns on ONE shared copy: RW serial read-modify-write rounds with a barrier each = ~8 us of the 19 us
  // the B = 4096 case took; shared-memory atomics were worse still, ~17 us.)
  {
    float* mine = part + (size_t)(threadIdx.x >> 5) * (L + 1) * d;
#pragma unroll
    for (int kk = 0; kk < N; ++kk) {
      const int i = (kk * 32 + lane) * 4;
      if (i < d) {
        *reinterpret_cast<float4*>(mine + (size_t)L * d + i) =
            make_float4(acc_g[kk * 4 + 0], acc_g[kk * 4 + 1], acc_g[kk * 4 + 2], acc_g[kk * 4 + 3]);
#pragma unroll
        for (int l = 0; l < LM; ++l) {
          if (l < L)
            *reinterpret_cast<float4*>(mine + (size_t)l * d + i) =
                make_float4(acc_a[l][kk * 4 + 0], acc_a[l][kk * 4 + 1], acc_a[l][kk * 4 + 2], acc_a[l][kk * 4 + 3]);
        }
      }
    }
    if (lane == 0) {
#pragma unroll
      for (int l = 0; l < LM; ++l) partT[(threadIdx.x >> 5) * LM + l] = T[l];     // T is warp-uniform
    }
  }
  __syncthreads();
  float Tl[LM];
#pragma unroll
  for (int l = 0; l < LM; ++l) {
    Tl[l] = 0.f;
    for (int wv = 0; wv < RW; ++wv) Tl[l] += partT[wv * LM + l];
  }
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    float G = 0.f, A[LM];
#pragma unroll
    for (int l = 0; l < LM; ++l) A[l] = 0.f;
    for (int wv = 0; wv < RW; ++wv) {
      const float* src = part + (size_t)wv * (L + 1) * d + i;
      G += src[(size_t)L * d];
#pragma unroll
      for (int l = 0; l < LM; ++l)
        if (l < L) A[l] += src[(size_t)l * d];
    }
    float cb = 0.f, wsum = 0.f;                      // cb_l = sum_{k<l} b_k ; wsum = sum_{k>l} w_k*T_k built from the top
    float dbv[LM];
#pragma unroll
    for (int l = LM - 1; l >= 0; --l) {
      dbv[l] = 0.f;
      if (l < L) { dbv[l] = G + wsum; wsum += sw[(size_t)l * d + i] * Tl[l]; }
    }
#pragma unroll
    for (int l = 0; l < LM; ++l) {
      if (l < L) {
        atomicAdd(dw + (size_t)l * d + i, A[l] + cb * Tl[l]);
        atomicAdd(db + (size_t)l * d + i, dbv[l]);
        cb += sb[(size_t)l * d + i];
      }
    }
  }
}

// Forward FUSED with the lookup (DCN/dcn.py:153-160: net = input_layer(...); x_{l+1} = cross_layer(x0, x_l, l)): the warp that owns a
// sample gathers its F table rows straight into the registers that hold x0, writes x0 once (the backward needs it) and runs the
// stack in the scalar-recurrence form of cross_bwd_reg_kernel -- x_l = x0 (1 + cs_l) + cb_l, so the L dot products u_l = x0 . w_l
// are independent (one batched butterfly) and  out = x0 (1 + cs_L) + cb_L.  Shared memory holds w, cb_L and the L scalars
// v_l = cb_l . w_l (computed once per CTA by warp 0); ~90 registers keep 2-3 CTAs per SM, which is what a 4096-sample batch
// needs (the register-resident-parameter version ran 1 CTA/SM and was slower than two launches).
// ids < 0 or >= the field's row count give the zero vector, exactly like ctr_embed_fm2_fwd.
template <int N, int LM, typename IdT>
__global__ void __launch_bounds__(CROSS_WARPS * 32)
embed_cross_fwd_kernel(const float* __restrict__ table, const long long* __restrict__ off, const IdT* __restrict__ ids,
                       const float* __restrict__ w, const float* __restrict__ b, int B, int F, int D, int L,
                       float* __restrict__ x0_out, float* __restrict__ out) {
  constexpr int NV = N * 4;
  extern __shared__ __align__(16) float smem[];
  const int d = F * D;
  float* sw = smem;                          // (L, d)
  float* scb = sw + (size_t)L * d;           // (d)   cb_L = sum_l b_l
  float* svl = scb + d;                      // (LM)  v_l = cb_l . w_l
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < L * d; i += blockDim.x) sw[i] = __ldg(w + i);
  if (threadIdx.x < 32) {                    // warp 0: prefix biases and the L scalars (reads w from global: no barrier needed)
    float cb[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) cb[k] = 0.f;
#pragma unroll
    for (int l = 0; l < LM; ++l) {
      if (l < L) {
        float dot = 0.f;
#pragma unroll
        for (int k = 0; k < N; ++k) {
          const int i = (k * 32 + lane) * 4;
          if (i < d) {
            const float4 tw = __ldg(reinterpret_cast<const float4*>(w + (size_t)l * d + i));
            const float4 tb = __ldg(reinterpret_cast<const float4*>(b + (size_t)l * d + i));
            dot += cb[k * 4 + 0] * tw.x + cb[k * 4 + 1] * tw.y + cb[k * 4 + 2] * tw.z + cb[k * 4 + 3] * tw.w;
            cb[k * 4 + 0] += tb.x; cb[k * 4 + 1] += tb.y; cb[k * 4 + 2] += tb.z; cb[k * 4 + 3] += tb.w;
          }
        }
        dot = warp_sum(dot);
        if (lane == 0) svl[l] = dot;
      }
    }
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const int i = (k * 32 + lane) * 4;
      if (i < d) *reinterpret_cast<float4*>(scb + i) = make_float4(cb[k * 4], cb[k * 4 + 1], cb[k * 4 + 2], cb[k * 4 + 3]);
    }
  }
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  int fk[N], part[N];
#pragma unroll
  for (int k = 0; k < N; ++k) {
    const int i = (k * 32 + lane) * 4;
    fk[k] = i < d ? i / D : -1;
    part[k] = i < d ? i - fk[k] * D : 0;
  }
  auto gather = [&](int s, float (&a)[NV]) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
      if (fk[k] >= 0) {
        const long long id = (long long)__ldg(ids + (size_t)s * F + fk[k]);
        const long long base = __ldg(off + fk[k]);
        if (id >= 0 && id < __ldg(off + fk[k] + 1) - base)
          t = __ldg(reinterpret_cast<const float4*>(table + (size_t)(base + id) * D + part[k]));
      }
      a[k * 4 + 0] = t.x; a[k * 4 + 1] = t.y; a[k * 4 + 2] = t.z; a[k * 4 + 3] = t.w;
    }
  };
  float na[NV];
  if (warp0 < B) gather(warp0, na);          // in flight while the parameters are staged
  __syncthreads();
  for (int s = warp0; s < B; s += nwarps) {
    float a0[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) a0[k] = na[k];
    if (s + nwarps < B) gather(s + nwarps, na);
    float red[LM];
#pragma unroll
    for (int l = 0; l < LM; ++l) {
      red[l] = 0.f;
      if (l < L) {
        float wv[NV];
        lane_load_smem<4, N>(wv, sw + (size_t)l * d, d, lane);
#pragma unroll
        for (int k = 0; k < NV; ++k) red[l] += a0[k] * wv[k];
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int l = 0; l < LM; ++l) red[l] += __shfl_xor_sync(0xffffffffu, red[l], o);
    }
    float cs = 0.f;
#pragma unroll
    for (int l = 0; l < LM; ++l)
      if (l < L) cs += (1.f + cs) * red[l] + svl[l];
    const float scale = 1.f + cs;
#pragma unroll
    for (int k = 0; k < N; ++k) {
      const int i = (k * 32 + lane) * 4;
      if (i < d) {
        const float4 cb = *reinterpret_cast<const float4*>(scb + i);
        *reinterpret_cast<float4*>(x0_out + (size_t)s * d + i) = make_float4(a0[k * 4], a0[k * 4 + 1], a0[k * 4 + 2], a0[k * 4 + 3]);
        *reinterpret_cast<float4*>(out + (size_t)s * d + i) =
            make_float4(a0[k * 4] * scale + cb.x, a0[k * 4 + 1] * scale + cb.y, a0[k * 4 + 2] * scale + cb.z, a0[k * 4 + 3] * scale + cb.w);
      }
    }
  }
}

static size_t cross_bwd_smem(int64_t d, int64_t L, bool has_xl, bool prefetch) {
  return sizeof(float) * ((size_t)3 * L * d + (size_t)(prefetch ? 2 : 1) * (has_xl ? 3 : 2) * CROSS_WARPS * d +
                          2 * CROSS_WARPS * CROSS_LMAX);     // sized for the larger layer bound
}

template <int VEC, int N>
static int launch_cross_fwd(const float* x0, const float* xl_in, const float* w, const float* b, int64_t B, int64_t d,
                            int64_t L, float* out, cudaStream_t st) {
  auto k = cross_fwd_kernel<VEC, N>;
  const size_t smem = sizeof(float) * 2 * (size_t)L * d;
  if (smem > 48 * 1024) CTR_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, CROSS_WARPS * 32, smem);
  if (per_sm < 1) per_sm = 1;
  long long grid = (long long)per_sm * sm_count();
  const long long need = (B + CROSS_WARPS - 1) / CROSS_WARPS;
  if (grid > need) grid = need;
  k<<<(int)grid, CROSS_WARPS * 32, smem, st>>>(x0, xl_in, w, b, (int)B, (int)d, (int)L, out);
  CTR_CHECK_LAUNCH("ctr_cross_fwd");
  return CTR_OK;
}

template <int VEC, int N, int CPT>
static int launch_cross_bwd(const float* x0, const float* xl_in, const float* w, const float* b, const float* g,
                            int64_t B, int64_t d, int64_t L, float* dx0, float* dxl, float* dw, float* db,
                            cudaStream_t st) {
  if constexpr (VEC == 4 && N <= 4) {                  // d <= 512: the lane-owned accumulators fit the register file
    if (xl_in == nullptr && L <= 4) {                  // the chain every reference model builds (DCN/dcn.py:157-160)
      // 12 warps per CTA (168 registers each) once all of them have work (two samples each): one sample of prefetch per warp is
      // then ~46 KB in flight per SM, and a 4096-sample batch is 2.3 instead of 3.5 dependent samples per warp.  (N = 4, L = 4
      // would spill at 168 registers.)
      const bool wide = B >= (int64_t)sm_count() * 12 * 2 && !(N == 4 && L > 3);
      const int rw = wide ? 12 : 8;
      const size_t smem_r = sizeof(float) * ((size_t)2 * L * d + (size_t)rw * ((L + 1) * d + 4));
      if (smem_r <= 200 * 1024) {
        auto pick = [&](auto tag) {
          constexpr int RW = decltype(tag)::value;
          return L <= 1 ? cross_bwd_reg_kernel<N, 1, RW> : L == 2 ? cross_bwd_reg_kernel<N, 2, RW>
               : L == 3 ? cross_bwd_reg_kernel<N, 3, RW> : cross_bwd_reg_kernel<N, 4, RW>;
        };
        auto kr = wide ? pick(std::integral_constant<int, 12>{}) : pick(std::integral_constant<int, 8>{});
        if (smem_r > 48 * 1024) CTR_CUDA(cudaFuncSetAttribute(kr, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_r));
        int per_sm = 1;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kr, rw * 32, smem_r);
        if (per_sm < 1) per_sm = 1;
        long long grid = (long long)per_sm * sm_count();
        const long long need = (B + rw - 1) / rw;
        if (grid > need) grid = need;
        if (db == dw + L * d) {                          // the host API allocates dw | db back to back: one memset node
          CTR_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * 2 * L * d, st));
        } else {
          CTR_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * L * d, st));
          CTR_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * L * d, st));
        }
        kr<<<(int)grid, rw * 32, smem_r, st>>>(x0, w, b, g, (int)B, (int)d, (int)L, dx0, dw, db);
        CTR_CHECK_LAUNCH("ctr_cross_bwd");
        return CTR_OK;
      }
    }
  }
  // double-buffered cp.async staging needs 16-byte rows (VEC == 4) and has to fit next to the parameter tables
  const bool pf = VEC == 4 && cross_bwd_smem(d, L, xl_in != nullptr, true) <= 160 * 1024;
  // LM = compile-time bound of the unrolled layer loops (predicated-off iterations still issue): 4 covers the reference's sweeps
  auto k = L <= 4 ? (pf ? cross_bwd_kernel<VEC, N, CPT, VEC == 4, 4> : cross_bwd_kernel<VEC, N, CPT, false, 4>)
                  : (pf ? cross_bwd_kernel<VEC, N, CPT, VEC == 4, 8> : cross_bwd_kernel<VEC, N, CPT, false, 8>);
  const size_t smem = cross_bwd_smem(d, L, xl_in != nullptr, pf);
  if (smem > 48 * 1024) CTR_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, CROSS_WARPS * 32, smem);
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 2) per_sm = 2;                         // fewer CTAs -> fewer atomic merges of dw/db
  long long grid = (long long)per_sm * sm_count();
  const long long need = (B + CROSS_WARPS - 1) / CROSS_WARPS;
  if (grid > need) grid = need;
  CTR_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * L * d, st));
  CTR_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * L * d, st));
  k<<<(int)grid, CROSS_WARPS * 32, smem, st>>>(x0, xl_in, w, b, g, (int)B, (int)d, (int)L, dx0, dxl, dw, db);
  CTR_CHECK_LAUNCH("ctr_cross_bwd");
  return CTR_OK;
}

}  // namespace ctr

using namespace ctr;

// d is served by N element groups per lane: vector path (VEC=4) when d % 4 == 0, scalar path otherwise.
#define CTR_CROSS_DISPATCH(FN, ...)                                                          \
  if (d % 4 == 0) {                                                                          \
    const int64_t n = (d / 4 + 31) / 32;                                                     \
    if (n <= 1) return FN(4, 1, __VA_ARGS__);                                                \
    if (n <= 2) return FN(4, 2, __VA_ARGS__);                                                \
    if (n <= 4) return FN(4, 4, __VA_ARGS__);                                                \
    return FN(4, 8, __VA_ARGS__);                                                            \
  } else {                                                                                   \
    const int64_t n = (d + 31) / 32;                                                         \
    if (n <= 1) return FN(1, 1, __VA_ARGS__);                                                \
    if (n <= 2) return FN(1, 2, __VA_ARGS__);                                                \
    if (n <= 4) return FN(1, 4, __VA_ARGS__);                                                \
    if (n <= 8) return FN(1, 8, __VA_ARGS__);                                                \
    if (n <= 16) return FN(1, 16, __VA_ARGS__);                                              \
    return FN(1, 32, __VA_ARGS__);                                                           \
  }

static int check_cross(const char* fn, int64_t B, int64_t d, int64_t L) {
  CTR_REQUIRE(B >= 0 && d >= 1 && L >= 1, "%s: bad sizes B=%lld d=%lld L=%lld", fn, (long long)B, (long long)d,
              (long long)L);
  CTR_UNSUPPORTED(d > 1024, "%s: d=%lld > 1024 unsupported", fn, (long long)d);
  CTR_UNSUPPORTED(L > CROSS_LMAX, "%s: L=%lld > %d unsupported", fn, (long long)L, CROSS_LMAX);
  return CTR_OK;
}

extern "C" int ctr_cross_fwd(const float* x0, const float* xl_in, const float* w, const float* b, int64_t B, int64_t d,
                             int64_t L, float* out, void* stream) {
  int rc = check_cross("ctr_cross_fwd", B, d, L);
  if (rc) return rc;
  CTR_REQUIRE(x0 && w && b && out, "ctr_cross_fwd: null argument");
  if (d % 4 == 0)
    CTR_REQUIRE(aligned16(x0) && aligned16(xl_in) && aligned16(out), "ctr_cross_fwd: buffers must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
#define FWD(V, NN, ...) launch_cross_fwd<V, NN>(__VA_ARGS__)
  CTR_CROSS_DISPATCH(FWD, x0, xl_in, w, b, B, d, L, out, st)
#undef FWD
}

extern "C" int ctr_cross_bwd(const float* x0, const float* xl_in, const float* w, const float* b, const float* g_out,
                             int64_t B, int64_t d, int64_t L, float* dx0, float* dxl_in, float* dw, float* db,
                             void* stream) {
  int rc = check_cross("ctr_cross_bwd", B, d, L);
  if (rc) return rc;
  CTR_REQUIRE(x0 && w && b && g_out && dx0 && dw && db, "ctr_cross_bwd: null argument");
  CTR_REQUIRE((xl_in == nullptr) == (dxl_in == nullptr), "ctr_cross_bwd: xl_in and dxl_in must both be given or both NULL");
  if (d % 4 == 0)
    CTR_REQUIRE(aligned16(x0) && aligned16(xl_in) && aligned16(g_out) && aligned16(dx0) && aligned16(dxl_in),
                "ctr_cross_bwd: buffers must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  if (B == 0) {
    CTR_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * L * d, st));
    CTR_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * L * d, st));
    return CTR_OK;
  }
#define BWD(V, NN, ...)                                                        \
  (d <= 256 ? launch_cross_bwd<V, NN, 1>(__VA_ARGS__)                          \
            : d <= 512 ? launch_cross_bwd<V, NN, 2>(__VA_ARGS__) : launch_cross_bwd<V, NN, 4>(__VA_ARGS__))
  CTR_CROSS_DISPATCH(BWD, x0, xl_in, w, b, g_out, B, d, L, dx0, dxl_in, dw, db, st)
#undef BWD
}

template <int N, typename IdT>
static int launch_embed_cross(const float* table, const int64_t* off, const IdT* ids, const float* w, const float* b, int64_t B,
                              int64_t F, int64_t D, int64_t L, float* x0, float* out, cudaStream_t st) {
  auto k = L <= 1 ? embed_cross_fwd_kernel<N, 1, IdT> : L == 2 ? embed_cross_fwd_kernel<N, 2, IdT>
         : L == 3 ? embed_cross_fwd_kernel<N, 3, IdT> : embed_cross_fwd_kernel<N, 4, IdT>;
  const size_t smem = sizeof(float) * ((size_t)L * F * D + F * D + 8);
  int per_sm = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, CROSS_WARPS * 32, smem);
  if (per_sm < 1) per_sm = 1;
  long long grid = (long long)per_sm * sm_count();
  const long long need = (B + CROSS_WARPS - 1) / CROSS_WARPS;
  if (grid > need) grid = need;
  k<<<(int)grid, CROSS_WARPS * 32, smem, st>>>(table, reinterpret_cast<const long long*>(off), ids, w, b, (int)B, (int)F, (int)D,
                                             (int)L, x0, out);
  CTR_CHECK_LAUNCH("ctr_embed_cross_fwd");
  return CTR_OK;
}

extern "C" int ctr_embed_cross_fwd(const float* table, const int64_t* field_row_offset, const void* ids, int ids_are_int32,
                                   int64_t B, int64_t F, int64_t D, const float* w, const float* b, int64_t L, float* x0,
                                   float* out, void* stream) {
  CTR_REQUIRE(B >= 0 && F >= 1 && D >= 1 && L >= 1, "ctr_embed_cross_fwd: bad sizes B=%lld F=%lld D=%lld L=%lld", (long long)B,
              (long long)F, (long long)D, (long long)L);
  CTR_REQUIRE(table && field_row_offset && ids && w && b && x0 && out, "ctr_embed_cross_fwd: null argument");
  const int64_t d = F * D;
  CTR_UNSUPPORTED((D & 3) != 0 || d > 512 || L > 4, "ctr_embed_cross_fwd: needs D %% 4 == 0, F*D <= 512, L <= 4 (D=%lld, d=%lld, "
                  "L=%lld); use ctr_embed_fm2_fwd + ctr_cross_fwd", (long long)D, (long long)d, (long long)L);
  CTR_REQUIRE(aligned16(table) && aligned16(w) && aligned16(b) && aligned16(x0) && aligned16(out),
              "ctr_embed_cross_fwd: arrays must be 16-byte aligned");
  CTR_REQUIRE(B < (1ll << 31), "ctr_embed_cross_fwd: batch too large");
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  const int n = (int)((d + 127) / 128);
#define EC(NN)                                                                                                              \
  return ids_are_int32 ? launch_embed_cross<NN, int>(table, field_row_offset, static_cast<const int*>(ids), w, b, B, F, D, L, x0, \
                                                     out, st)                                                                \
                       : launch_embed_cross<NN, long long>(table, field_row_offset, static_cast<const long long*>(ids), w, b, B, \
                                                           F, D, L, x0, out, st);
  if (n <= 1) { EC(1) } else if (n == 2) { EC(2) } else if (n == 3) { EC(3) } else { EC(4) }
#undef EC
}


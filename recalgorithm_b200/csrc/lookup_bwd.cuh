// The config-5 lookup backward, row_grads[b,f,:] = d_tile[b,f,:] + g[b] * (S[b,:] - e[b,f,:]) with S[b,:] = sum_f e[b,f,:],
// written once for every kernel that computes it: the plain / BI / LIN backward (embed_fm2.cu), the backward fused with
// the gradient exchange (sharded.cu) and the backward fused with the sparse Adam step (adam.cu).
//
// One warp per sample.  Chunk j of the sample's n4 = F*LPR float4 belongs to lane j % 32, and its embedding chunk is
// j % LPR == lane % LPR, so the lanes that share a chunk are LPR apart.  With HOLD > 0 the sample's tile row stays in
// registers (HOLD float4 per lane, F*D <= HOLD*128 floats) between the S pass and the gradient pass; HOLD == 0 is the
// two-pass form for wider rows (the second pass re-reads the row through L1/L2).
#pragma once
#include "ctr_common.cuh"

namespace ctr {

__device__ __forceinline__ float4 f4_zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }

// A per-field id of the fused lookups: int64 (TF's sparse ids) or int32 (half the bytes of the id matrix), read once.
__device__ __forceinline__ long long load_id(const long long* p) { return ldg_stream_i64(p); }
__device__ __forceinline__ long long load_id(const int* p) {
  int r;
  asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(r) : "l"(p));
  return (long long)r;
}

// completes a per-lane partial sum over the lanes that hold the same chunk
template <int LPR>
__device__ __forceinline__ void lane_group_sum(float4& v) {
#pragma unroll
  for (int o = LPR; o < 32; o <<= 1) {
    v.x += __shfl_xor_sync(0xffffffffu, v.x, o); v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
    v.z += __shfl_xor_sync(0xffffffffu, v.z, o); v.w += __shfl_xor_sync(0xffffffffu, v.w, o);
  }
}

// one finished chunk: dt + g * (S - e)
__device__ __forceinline__ float4 fm2_row_grad(const float4& dt, const float4& g, const float4& S, const float4& e) {
  float4 r;
  r.x = dt.x + g.x * (S.x - e.x); r.y = dt.y + g.y * (S.y - e.y);
  r.z = dt.z + g.z * (S.z - e.z); r.w = dt.w + g.w * (S.w - e.w);
  return r;
}

// Streams the sample's tile row into registers, e[k] = e_row[k*32 + lane] (zero past n4); `chunk(k, j)` runs after
// each in-range chunk's load has issued.
template <int HOLD, class Chunk>
__device__ __forceinline__ void load_tile_row(float4 (&e)[HOLD], const float4* __restrict__ e_row, int n4, int lane, Chunk&& chunk) {
#pragma unroll
  for (int k = 0; k < HOLD; ++k) {
    const int j = k * 32 + lane;
    e[k] = f4_zero();
    if (j < n4) {
      e[k] = ldg_f4(e_row + j);
      chunk(k, j);
    }
  }
}

// S of the register-held row, complete in every lane
template <int LPR, int HOLD>
__device__ __forceinline__ float4 tile_row_sum(const float4 (&e)[HOLD]) {
  float4 S = f4_zero();
#pragma unroll
  for (int k = 0; k < HOLD; ++k) { S.x += e[k].x; S.y += e[k].y; S.z += e[k].z; S.w += e[k].w; }
  lane_group_sum<LPR>(S);
  return S;
}

// Upstream gradient d_tile of a sample (the `head` of lookup_bwd_sample): `load(d, j)` issues with the tile loads, before
// the S reduction, into d (zero on entry); `at(j, d)` is the term at use; `add(k, e)` sees every finished chunk.
// RowGrad: d_tile is a (B, F, D) tensor; its rows are streamed (none: d_tile == nullptr, the term is zero).
struct RowGrad {
  const float4* __restrict__ row;
  __device__ __forceinline__ void load(float4& d, int j) const {
    if (row != nullptr) d = ldg_f4(row + j);
  }
  __device__ __forceinline__ float4 at(int, const float4& d) const { return d; }
  __device__ __forceinline__ void add(int, const float4&) {}
};

// LinHead: a dense(1) consumer of the flattened tile is fused in (ctr_embed_fm2_lin_fwd), so d_tile is the rank-1
// product d_lin[b] * wlin[f,d] and is never materialised: it is formed at use from wlin in shared memory, and
// d_wlin = sum_b d_lin[b] * e[b] is accumulated in registers (HOLD float4 per lane), then per CTA one shared-memory
// reduction and one vector red.global.add per element.  Needs 2 * n4 float4 of dynamic shared memory.
template <int HOLD>
struct LinHead {
  static_assert(HOLD > 0, "the LIN head needs the register-resident row");
  float4* s_w;          // [n4] wlin, then [n4] d_wlin accumulator
  int n4;
  float gl;             // d_lin of the current sample
  float4 acc[HOLD];
  __device__ __forceinline__ void stage(float4* smem, const float4* __restrict__ wlin, int n) {
    s_w = smem;
    n4 = n;
    for (int j = threadIdx.x; j < n4; j += blockDim.x) { s_w[j] = __ldg(wlin + j); s_w[n4 + j] = f4_zero(); }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < HOLD; ++k) acc[k] = f4_zero();
  }
  __device__ __forceinline__ void load(float4&, int) const {}
  __device__ __forceinline__ float4 at(int j, const float4&) const {
    const float4 w = s_w[j];
    return make_float4(gl * w.x, gl * w.y, gl * w.z, gl * w.w);
  }
  __device__ __forceinline__ void add(int k, const float4& e) {
    acc[k].x += gl * e.x; acc[k].y += gl * e.y; acc[k].z += gl * e.z; acc[k].w += gl * e.w;
  }
  __device__ __forceinline__ void flush(float4* __restrict__ d_wlin, int lane) {
#pragma unroll
    for (int k = 0; k < HOLD; ++k) {
      const int j = k * 32 + lane;
      if (j < n4) {
        float* a = reinterpret_cast<float*>(s_w + n4 + j);
        atomicAdd(a + 0, acc[k].x); atomicAdd(a + 1, acc[k].y); atomicAdd(a + 2, acc[k].z); atomicAdd(a + 3, acc[k].w);
      }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < n4; j += blockDim.x) atomicAdd(d_wlin + j, s_w[n4 + j]);
  }
};

// The backward of one sample.  `g` is d_fm2[b] in every component, or the (D,) gradient of the BI vector (this lane's
// chunk).  The sink takes the finished chunks: `fetch(k, j)` runs with the d_tile loads (HOLD > 0 only) and may load
// per-chunk state, `sink(k, j, r)` receives r = row_grads[b] chunk j (k is its register slot; 0 in the two-pass form).
template <int LPR, int HOLD, class Head, class Sink>
__device__ __forceinline__ void lookup_bwd_sample(const float4* __restrict__ e_row, int n4, int lane, const float4& g, Head& head,
                                                  Sink& sink) {
  if constexpr (HOLD > 0) {
    float4 e[HOLD], dt[HOLD];
    load_tile_row(e, e_row, n4, lane, [](int, int) {});
#pragma unroll
    for (int k = 0; k < HOLD; ++k) {
      const int j = k * 32 + lane;
      dt[k] = f4_zero();
      if (j < n4) {
        head.load(dt[k], j);
        sink.fetch(k, j);
      }
    }
    const float4 S = tile_row_sum<LPR>(e);
#pragma unroll
    for (int k = 0; k < HOLD; ++k) {
      const int j = k * 32 + lane;
      if (j < n4) {
        sink(k, j, fm2_row_grad(head.at(j, dt[k]), g, S, e[k]));
        head.add(k, e[k]);
      }
    }
  } else {
    float4 S = f4_zero();
    for (int j = lane; j < n4; j += 32) {
      const float4 v = __ldg(e_row + j);
      S.x += v.x; S.y += v.y; S.z += v.z; S.w += v.w;
    }
    lane_group_sum<LPR>(S);
    for (int j = lane; j < n4; j += 32) {
      const float4 v = __ldg(e_row + j);
      float4 dt = f4_zero();
      head.load(dt, j);
      sink(0, j, fm2_row_grad(head.at(j, dt), g, S, v));
    }
  }
}

// Host side: the (B, F, D) bounds of the fused 128-bit row kernels, checked by every entry point `fn` that launches one.
static int check_bfd(const char* fn, int64_t B, int64_t F, int64_t D) {
  CTR_REQUIRE(B >= 0 && F >= 1 && D >= 1, "%s: bad sizes B=%lld F=%lld D=%lld", fn, (long long)B, (long long)F,
              (long long)D);
  CTR_REQUIRE(B <= 0x7fffffffLL / 8 && F <= 65536, "%s: B=%lld / F=%lld too large", fn, (long long)B, (long long)F);
  CTR_UNSUPPORTED(D % 4 != 0 || D > 128 || (D & (D - 1)) != 0,
                  "%s: D=%lld unsupported by the fused 128-bit path (need a power of two in 4..128); "
                  "use ctr_bag_lookup_* for other widths", fn, (long long)D);
  return CTR_OK;
}

// Host side: the HOLD of a sample of F fields of LPR chunks, from its ceil(F*LPR/32) chunks per lane: 4, 8 or 12.  Above
// 12 (F*D > 1536) a kernel with the two-pass form takes HOLD = 0; any other fails with CTR_ERR_UNSUPPORTED, naming the
// entry point `fn` and appending `hint` to the message.
template <bool TWO_PASS, class Fn>
int with_hold(int64_t F, int64_t LPR, Fn&& f, const char* fn = "", const char* hint = "") {
  const int64_t per_lane = (F * LPR + 31) / 32;
  if (per_lane <= 4) return f(std::integral_constant<int, 4>{});
  if (per_lane <= 8) return f(std::integral_constant<int, 8>{});
  if (per_lane <= 12) return f(std::integral_constant<int, 12>{});
  if constexpr (TWO_PASS) {
    return f(std::integral_constant<int, 0>{});
  } else {
    set_error("%s: F*D = %lld exceeds the register-resident limit of 1536%s", fn, (long long)(F * LPR * 4), hint);
    return CTR_ERR_UNSUPPORTED;
  }
}

}  // namespace ctr

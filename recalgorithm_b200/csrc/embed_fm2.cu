// Row L + Row FM2 (SURVEY.md section 8a): fused per-field embedding lookup + DeepFM second-order term.
//
// Reference semantics being replaced (paths relative to the reference's algorithm/ directory):
//   * fc.input_layer(features, [embedding_column]) once per field  -- DeepFM/deepfm.py:187-190
//     (row gather; pruned id -> zero vector; TF-internal, SURVEY A.5)
//   * square(add_n(e)), add_n(square(e)), reduce_sum(0.5*(a-b), axis=1) -- DeepFM/deepfm.py:192-200
//   * the gather's IndexedSlices gradient + d(FM2)/d(e) = g*(S - e)
//
// H100 mapping (HBM-bound gather; no tensor cores):
//   one warp per sample; a row of D fp32 is LPR = D/4 lanes x 128-bit, so one warp-level LDG.128
//   fetches RPW = 32/LPR complete rows (D=32: 4 rows x 128 B = 4 full cache lines).  The ids of up
//   to 32 fields are read with ONE coalesced 8-byte load per lane and distributed by shuffle, so all
//   row addresses of a sample are known before the first row load issues -> up to 8 independent
//   128-bit loads in flight per lane (enough outstanding bytes per SM to cover HBM latency).
//   S = sum_f e and Q = sum_f e^2 accumulate in registers; the FM2 logit is a shuffle reduction.
//   The (B,F,D) tile is written with plain stores: its last-written rows are still in L2 when the backward, which walks the
//   samples from the last one down, reads them first.
#include "lookup_bwd.cuh"

namespace ctr {

// Row-sharded tables (SURVEY 8e): global row gr lives on rank gr % G at local row gr / G (G a power of two <= 8).
// `base[r]` is rank r's shard as seen from THIS GPU (peer-mapped over NVLink for r != my rank), so the gather pulls
// remote rows with the same 128-bit loads and the return all-to-all disappears into the kernel.
struct PeerTables {
  const float4* base[8];
  int G, logG;
};

// BI: `fm2` points at a (B, D) buffer that receives 0.5*(S^2 - Q) per embedding dim (NFM bi-interaction pooling,
// NFM/nfm.py:155-168) instead of its sum over D.
// IdT: int64 ids (TF's sparse ids) or int32 ids (half the PCIe / HBM bytes of the id matrix; `ids64_out`, when given,
// receives the widened copy that IndexedSlices consumers downstream expect).
// rows of a peer shard: plain (L1-allocating) loads -- measured 650 GB/s over NVLink against 622 GB/s for
// .nc.L1::no_allocate (tools/peerbench.cu); peer lines bypass the local L2 either way
__device__ __forceinline__ float4 ld_peer_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

// LIN: a dense(1) consumer of the flattened tile is fused in: lin[b] = sum_{f,d} e[b,f,d] * wlin[f,d] (the kernel of a
// tf.layers.dense(units=1, use_bias=False) over the (B, F*D) input_layer output), so the consumer never re-streams the tile.
// SEQ: every column of the id matrix indexes the SAME table (rows [row_off[0], row_off[1])): the (B, T) history of a sequence
// feature (sequence_input_layer over a shared embedding, DIN/din.py:209-214) gathered with one warp per sample instead of
// one per id.
template <int LPR, bool SH, int MINB, bool BI = false, typename IdT = long long, bool LIN = false, bool SEQ = false>
__global__ void __launch_bounds__(256, MINB)
embed_fm2_fwd_kernel(const float4* __restrict__ table, const PeerTables peers, const long long* __restrict__ row_off,
                     const IdT* __restrict__ ids, int B, int F, float4* __restrict__ tile,
                     float* __restrict__ fm2, long long* __restrict__ ids64_out,
                     const float4* __restrict__ wlin, float* __restrict__ lin) {
  constexpr int RPW = 32 / LPR;             // rows fetched per warp-level load
  constexpr int UB = LPR < 8 ? LPR : 8;     // loads batched before first use
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR;               // which of the RPW rows this lane works on
  const int c = lane % LPR;                 // which 128-bit chunk of the row
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;

  for (int b = warp0; b < B; b += nwarps) {
    float4 S = f4_zero(), Q = f4_zero();
    float lin_acc = 0.f;
    for (int f0 = 0; f0 < F; f0 += 32) {
      const int nf = min(32, F - f0);
      long long row = -1;
      if (lane < nf) {
        const long long id = load_id(ids + (size_t)b * F + f0 + lane);
        const long long lo = __ldg(row_off + (SEQ ? 0 : f0 + lane)), hi = __ldg(row_off + (SEQ ? 1 : f0 + lane + 1));
        row = (id >= 0 && id < hi - lo) ? lo + id : -1;      // OOV(-1)/out-of-range -> zero vector
        if (sizeof(IdT) == 4 && ids64_out != nullptr) ids64_out[(size_t)b * F + f0 + lane] = id;
      }
#pragma unroll
      for (int it0 = 0; it0 < LPR; it0 += UB) {              // LPR iterations cover 32 fields
        if (it0 * RPW >= nf) break;                           // warp-uniform
        float4 v[UB];
        bool in[UB];
#pragma unroll
        for (int u = 0; u < UB; ++u) {
          const int fs = (it0 + u) * RPW + sub;               // field slot inside this 32-chunk
          const long long r = __shfl_sync(full, row, fs);
          in[u] = fs < nf;
          v[u] = f4_zero();
          if (in[u] && r >= 0) {
            if (SH) v[u] = ld_peer_f4(peers.base[r & (peers.G - 1)] + (size_t)(r >> peers.logG) * LPR + c);
            else v[u] = ldg_f4(table + (size_t)r * LPR + c);
          }
        }
#pragma unroll
        for (int u = 0; u < UB; ++u) {
          S.x += v[u].x; S.y += v[u].y; S.z += v[u].z; S.w += v[u].w;
          // square THEN add, like tf.square + tf.add_n (no FMA contraction: keeps F == 1 exactly zero)
          Q.x = __fadd_rn(Q.x, __fmul_rn(v[u].x, v[u].x)); Q.y = __fadd_rn(Q.y, __fmul_rn(v[u].y, v[u].y));
          Q.z = __fadd_rn(Q.z, __fmul_rn(v[u].z, v[u].z)); Q.w = __fadd_rn(Q.w, __fmul_rn(v[u].w, v[u].w));
          if (tile != nullptr && in[u]) {
            const int fs = (it0 + u) * RPW + sub;
            tile[((size_t)b * F + f0 + fs) * LPR + c] = v[u];
          }
          if (LIN && in[u]) {
            const float4 w = __ldg(wlin + (size_t)(f0 + (it0 + u) * RPW + sub) * LPR + c);
            lin_acc += v[u].x * w.x + v[u].y * w.y + v[u].z * w.z + v[u].w * w.w;
          }
        }
      }
    }
    if (LIN) {
      lin_acc = warp_sum(lin_acc);
      if (lane == 0) lin[b] = lin_acc;
    }
    if (fm2 != nullptr) {
      // complete S and Q over the RPW row-groups (lanes sharing the same chunk c)
#pragma unroll
      for (int o = LPR; o < 32; o <<= 1) {
        S.x += __shfl_xor_sync(full, S.x, o); S.y += __shfl_xor_sync(full, S.y, o);
        S.z += __shfl_xor_sync(full, S.z, o); S.w += __shfl_xor_sync(full, S.w, o);
        Q.x += __shfl_xor_sync(full, Q.x, o); Q.y += __shfl_xor_sync(full, Q.y, o);
        Q.z += __shfl_xor_sync(full, Q.z, o); Q.w += __shfl_xor_sync(full, Q.w, o);
      }
      if (BI) {
        if (lane < LPR) {
          float4 r;
          r.x = 0.5f * __fsub_rn(__fmul_rn(S.x, S.x), Q.x); r.y = 0.5f * __fsub_rn(__fmul_rn(S.y, S.y), Q.y);
          r.z = 0.5f * __fsub_rn(__fmul_rn(S.z, S.z), Q.z); r.w = 0.5f * __fsub_rn(__fmul_rn(S.w, S.w), Q.w);
          reinterpret_cast<float4*>(fm2)[(size_t)b * LPR + c] = r;
        }
        continue;
      }
      // 0.5 * (S^2 - Q) per embedding dim, then reduce over D (4 components x LPR lanes)
      float p = 0.5f * __fsub_rn(__fmul_rn(S.x, S.x), Q.x) + 0.5f * __fsub_rn(__fmul_rn(S.y, S.y), Q.y) +
                0.5f * __fsub_rn(__fmul_rn(S.z, S.z), Q.z) + 0.5f * __fsub_rn(__fmul_rn(S.w, S.w), Q.w);
#pragma unroll
      for (int o = 1; o < LPR; o <<= 1) p += __shfl_xor_sync(full, p, o);
      if (lane == 0) fm2[b] = p;
    }
  }
}

// Backward: row_grads[b,f,:] = d_tile[b,f,:] + g[b] * (S[b,:] - e[b,f,:]), the per-sample body of lookup_bwd.cuh.
// FM2_BI: d_fm2 is the (B, D) gradient of the bi-interaction vector (g becomes per-dimension).
// FM2_LIN (HOLD > 0 only): the backward of the fused dense(1) head, d_tile carries wlin (F*D) and d_wlin = sum_b d_lin[b]*e[b]
// is accumulated (LinHead); row_grads[b,f,:] = d_lin[b]*wlin[f,:] + d_fm2[b]*(S[b,:] - e[b,f,:]).
enum { FM2_PLAIN, FM2_BI, FM2_LIN };

struct StoreRow {
  float4* __restrict__ o_row;
  __device__ __forceinline__ void fetch(int, int) {}
  __device__ __forceinline__ void operator()(int, int j, const float4& r) { stg_stream_f4(o_row + j, r); }
};

// LIN asks for 2 CTAs per SM; the plain and BI forms set no floor, so ptxas keeps their register count low.
template <int LPR, int HOLD, int MODE>
__global__ void __launch_bounds__(256, MODE == FM2_LIN ? 2 : 0)
embed_fm2_bwd_kernel(const float4* __restrict__ tile, const float4* __restrict__ d_tile, const float* __restrict__ d_fm2,
                     const float* __restrict__ d_lin, int B, int F, float4* __restrict__ row_grads, float4* __restrict__ d_wlin) {
  extern __shared__ float4 s_lin[];
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int n4 = F * LPR;
  LinHead<MODE == FM2_LIN ? HOLD : 1> lin;
  if (MODE == FM2_LIN) lin.stage(s_lin, d_tile, n4);
  for (int w = warp0; w < B; w += nwarps) {
    const int b = B - 1 - w;   // last sample first: the forward wrote it last, so its tile row is the likeliest L2 hit
    StoreRow sink{row_grads + (size_t)b * n4};
    RowGrad rows{d_tile ? d_tile + (size_t)b * n4 : nullptr};   // not read in LIN mode
    float4 g4;
    if (MODE == FM2_BI) {
      g4 = __ldg(reinterpret_cast<const float4*>(d_fm2) + (size_t)b * LPR + lane % LPR);
    } else {
      const float g = d_fm2 ? __ldg(d_fm2 + b) : 0.f;
      g4 = make_float4(g, g, g, g);
    }
    if constexpr (MODE == FM2_LIN) {
      lin.gl = d_lin ? __ldg(d_lin + b) : 0.f;
      lookup_bwd_sample<LPR, HOLD>(tile + (size_t)b * n4, n4, lane, g4, lin, sink);
    } else {
      lookup_bwd_sample<LPR, HOLD>(tile + (size_t)b * n4, n4, lane, g4, rows, sink);
    }
  }
  if (MODE == FM2_LIN) lin.flush(d_wlin, lane);
}

// grad_table[row(b,f), :] += row_grads[b,f,:]  (valid ids only) -- vector red.global.add.
template <int LPR>
__global__ void __launch_bounds__(256)
embed_scatter_add_kernel(float4* __restrict__ grad_table, const long long* __restrict__ row_off,
                         const long long* __restrict__ ids, const float4* __restrict__ row_grads, int B, int F) {
  const size_t total = (size_t)B * F * LPR;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % LPR);
    const size_t bf = t / LPR;
    const int f = (int)(bf % F);
    const long long id = __ldg(ids + bf);
    const long long lo = __ldg(row_off + f), hi = __ldg(row_off + f + 1);
    if (id >= 0 && id < hi - lo) {
      const float4 g = ldg_stream_f4(row_grads + t);
      atomicAdd(grad_table + (size_t)(lo + id) * LPR + c, g);
    }
  }
}

// ---- general multi-valued lookup (combiner='mean'), any D <= 256 ------------------------------------
// A group of G lanes (power of two, G >= min(D,32)) serves one bag; 32/G bags per warp.
__global__ void __launch_bounds__(256)
bag_lookup_fwd_kernel(const float* __restrict__ table, long long V, int D, const long long* __restrict__ ids,
                      const long long* __restrict__ offsets, int B, float* __restrict__ out, long long out_stride,
                      int G) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int gl = threadIdx.x % G;                     // lane inside the group
  const int nthreads = gridDim.x * blockDim.x;
  for (int b = tid / G; b < B; b += nthreads / G) {
    const long long s = __ldg(offsets + b), e = __ldg(offsets + b + 1);
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    int n = 0;
    for (long long i = s; i < e; ++i) {
      const long long id = __ldg(ids + i);
      if (id >= 0 && id < V) {
        ++n;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int dd = k * G + gl;
          if (dd < D) acc[k] += __ldg(table + (size_t)id * D + dd);
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int dd = k * G + gl;
      // mean = sum / count (TF divides the segment sum by the count); n == 0 -> zeros
      if (dd < D) out[(size_t)b * out_stride + dd] = n > 0 ? acc[k] / (float)n : 0.f;
    }
  }
}

__global__ void __launch_bounds__(256)
bag_lookup_bwd_kernel(const float* __restrict__ d_out, long long out_stride, long long V, int D,
                      const long long* __restrict__ ids, const long long* __restrict__ offsets, int B,
                      float* __restrict__ row_grads, int G) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int gl = threadIdx.x % G;
  const int nthreads = gridDim.x * blockDim.x;
  for (int b = tid / G; b < B; b += nthreads / G) {
    const long long s = __ldg(offsets + b), e = __ldg(offsets + b + 1);
    int n = 0;
    for (long long i = s; i < e; ++i) {
      const long long id = __ldg(ids + i);
      n += (id >= 0 && id < V);
    }
    for (long long i = s; i < e; ++i) {
      const long long id = __ldg(ids + i);
      const bool ok = id >= 0 && id < V;
      for (int dd = gl; dd < D; dd += G) {
        const float g = __ldg(d_out + (size_t)b * out_stride + dd);
        row_grads[(size_t)i * D + dd] = ok ? g / (float)n : 0.f;
      }
    }
  }
}

// ---- DeepFM first-order ("wide") term as a D=1 lookup (SURVEY 8f.1) --------------------------------------
// Reference: indicator_column multi-hot (B, sum V) @ dense(1) kernel (sum V, 1) + bias  (DeepFM/deepfm.py:72-80,180-181).
// A multi-hot times a one-column kernel is a per-id scalar gather-sum; id -1 contributes 0 (all-zero indicator row).
__global__ void __launch_bounds__(256)
first_order_fwd_kernel(const float* __restrict__ w, const long long* __restrict__ row_off,
                       const long long* __restrict__ ids, int B, int F, float bias, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int b = warp0; b < B; b += nwarps) {
    float acc = 0.f;
    for (int f = lane; f < F; f += 32) {
      const long long id = ldg_stream_i64(ids + (size_t)b * F + f);
      const long long lo = __ldg(row_off + f), hi = __ldg(row_off + f + 1);
      if (id >= 0 && id < hi - lo) acc += __ldg(w + lo + id);
    }
    acc = warp_sum(acc);
    if (lane == 0) out[b] = acc + bias;
  }
}

template <int LPR, typename IdT>
static int launch_fwd(const float* table, const PeerTables* peers, const int64_t* off, const IdT* ids, int64_t B,
                      int64_t F, float* tile, float* fm2, int64_t* ids64_out, cudaStream_t st) {
  PeerTables none = {};
  // 4 CTAs/SM (64 registers) measured 0.80 of HBM peak vs 0.71-0.80 uncapped; a next-sample id prefetch variant measured
  // neutral-to-negative (it costs spills) and was removed.  The sharded (peer-pull) variant keeps the register budget open.
  // The local gather runs one CTA per 8 samples instead of a resident grid: CTAs start in order, so the tile rows being
  // written at any moment stay in a narrow, advancing address range (1 % faster at config 5 on H100 SXM).
  const float4* table4 = reinterpret_cast<const float4*>(table);
  const long long* off64 = reinterpret_cast<const long long*>(off);
  float4* tile4 = reinterpret_cast<float4*>(tile);
  long long* ids64 = reinterpret_cast<long long*>(ids64_out);
  if (peers != nullptr)
    return launch_resident("ctr_embed_fm2_fwd", embed_fm2_fwd_kernel<LPR, true, 1, false, IdT>, (B + 7) / 8, 256, 0, st, table4,
                           *peers, off64, ids, (int)B, (int)F, tile4, fm2, ids64, nullptr, nullptr);
  return launch("ctr_embed_fm2_fwd", embed_fm2_fwd_kernel<LPR, false, 4, false, IdT>, (unsigned)((B + 7) / 8), 256, 0, st, table4,
                none, off64, ids, (int)B, (int)F, tile4, fm2, ids64, nullptr, nullptr);
}

// FM2_LIN has no two-pass form: wider rows fail in with_hold with `what` in the message.
// The plain and BI forms run one CTA per 8 samples (one sample per warp) instead of a resident grid: CTAs start in order, so
// the rows in flight stay in a narrow, advancing address range, which measured 2.5 % faster at config 5 on H100 SXM.  The LIN
// form stays resident: each CTA stages wlin and reduces its d_wlin once.
template <int MODE>
static int launch_bwd(const char* what, const float* tile, const float* d_tile, const float* d_fm2, const float* d_lin, int64_t B,
                      int64_t F, int64_t D, float* row_grads, float* d_wlin, cudaStream_t st) {
  return with_lpr(D, [&](auto LPR) {
    return with_hold<MODE != FM2_LIN>(F, LPR, [&](auto HOLD) {
      const auto k = embed_fm2_bwd_kernel<LPR, HOLD, MODE>;
      const float4* tile4 = reinterpret_cast<const float4*>(tile);
      const float4* d_tile4 = reinterpret_cast<const float4*>(d_tile);
      float4* row_grads4 = reinterpret_cast<float4*>(row_grads);
      float4* d_wlin4 = reinterpret_cast<float4*>(d_wlin);
      if (MODE != FM2_LIN)
        return launch(what, k, (unsigned)((B + 7) / 8), 256, 0, st, tile4, d_tile4, d_fm2, d_lin, (int)B, (int)F, row_grads4, d_wlin4);
      return launch_resident(what, k, (B + 7) / 8, 256, sizeof(float4) * 2 * (size_t)F * LPR, st, tile4, d_tile4, d_fm2, d_lin, (int)B,
                             (int)F, row_grads4, d_wlin4);
    }, what);
  });
}

template <int LPR>
static int launch_fwd_bi(const float* table, const int64_t* off, const int64_t* ids, int64_t B, int64_t F, float* tile,
                         float* bi, cudaStream_t st) {
  return launch_resident("ctr_embed_bi_fwd", embed_fm2_fwd_kernel<LPR, false, 4, true>, (B + 7) / 8, 256, 0, st,
                         reinterpret_cast<const float4*>(table), PeerTables{}, reinterpret_cast<const long long*>(off),
                         reinterpret_cast<const long long*>(ids), (int)B, (int)F, reinterpret_cast<float4*>(tile), bi, nullptr,
                         nullptr, nullptr);
}

template <typename IdT>
static int dispatch_fwd(const float* table, const PeerTables* peers, const int64_t* off, const IdT* ids, int64_t B,
                        int64_t F, int64_t D, float* tile, float* fm2, int64_t* ids64_out, cudaStream_t st) {
  return with_lpr(D, [&](auto LPR) { return launch_fwd<LPR>(table, peers, off, ids, B, F, tile, fm2, ids64_out, st); });
}

static int fill_peers(const char* fn, PeerTables& peers, const float* const* shard_ptrs, int64_t G) {
  CTR_REQUIRE(G >= 1 && G <= 8 && (G & (G - 1)) == 0, "%s: G=%lld must be a power of two <= 8", fn, (long long)G);
  peers = PeerTables{};
  peers.G = (int)G;
  while ((1 << peers.logG) < G) ++peers.logG;
  for (int r = 0; r < G; ++r) {
    CTR_REQUIRE(shard_ptrs[r] != nullptr && aligned16(shard_ptrs[r]), "%s: shard %d null/unaligned", fn, r);
    peers.base[r] = reinterpret_cast<const float4*>(shard_ptrs[r]);
  }
  return CTR_OK;
}

}  // namespace ctr

using namespace ctr;

extern "C" int ctr_embed_fm2_fwd(const float* table, const int64_t* field_row_offset, const int64_t* ids,
                                 int64_t B, int64_t F, int64_t D, float* tile, float* fm2, void* stream) {
  int rc = check_bfd("ctr_embed_fm2_fwd", B, F, D);
  if (rc) return rc;
  CTR_REQUIRE(table && field_row_offset && ids, "ctr_embed_fm2_fwd: null table/field_row_offset/ids");
  CTR_REQUIRE(tile || fm2, "ctr_embed_fm2_fwd: both outputs are NULL");
  CTR_REQUIRE(aligned16(table) && aligned16(tile), "ctr_embed_fm2_fwd: table and tile must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  return dispatch_fwd(table, nullptr, field_row_offset, reinterpret_cast<const long long*>(ids), B, F, D, tile, fm2, nullptr, st);
}

extern "C" int ctr_embed_fm2_fwd_ids32(const float* table, const int64_t* field_row_offset, const int32_t* ids, int64_t B,
                                       int64_t F, int64_t D, float* tile, float* fm2, int64_t* ids64_out, void* stream) {
  int rc = check_bfd("ctr_embed_fm2_fwd_ids32", B, F, D);
  if (rc) return rc;
  CTR_REQUIRE(table && field_row_offset && ids, "ctr_embed_fm2_fwd_ids32: null table/field_row_offset/ids");
  CTR_REQUIRE(tile || fm2, "ctr_embed_fm2_fwd_ids32: both outputs are NULL");
  CTR_REQUIRE(aligned16(table) && aligned16(tile), "ctr_embed_fm2_fwd_ids32: table and tile must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  return dispatch_fwd(table, nullptr, field_row_offset, reinterpret_cast<const int*>(ids), B, F, D, tile, fm2, ids64_out,
                      as_stream(stream));
}

extern "C" int ctr_embed_fm2_fwd_sharded(const float* const* shard_ptrs, int64_t G, const int64_t* field_row_offset,
                                         const int64_t* ids, int64_t B, int64_t F, int64_t D, float* tile, float* fm2,
                                         void* stream) {
  int rc = check_bfd("ctr_embed_fm2_fwd_sharded", B, F, D);
  if (rc) return rc;
  CTR_REQUIRE(shard_ptrs && field_row_offset && ids, "ctr_embed_fm2_fwd_sharded: null shard_ptrs/field_row_offset/ids");
  CTR_REQUIRE(tile || fm2, "ctr_embed_fm2_fwd_sharded: both outputs are NULL");
  PeerTables peers;
  rc = fill_peers("ctr_embed_fm2_fwd_sharded", peers, shard_ptrs, G);
  if (rc) return rc;
  CTR_REQUIRE(aligned16(tile), "ctr_embed_fm2_fwd_sharded: tile must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  return dispatch_fwd(nullptr, &peers, field_row_offset, reinterpret_cast<const long long*>(ids), B, F, D, tile, fm2, nullptr,
                      as_stream(stream));
}

extern "C" int ctr_embed_fm2_fwd_sharded_ids32(const float* const* shard_ptrs, int64_t G, const int64_t* field_row_offset,
                                               const int32_t* ids, int64_t B, int64_t F, int64_t D, float* tile, float* fm2,
                                               int64_t* ids64_out, void* stream) {
  int rc = check_bfd("ctr_embed_fm2_fwd_sharded_ids32", B, F, D);
  if (rc) return rc;
  CTR_REQUIRE(shard_ptrs && field_row_offset && ids, "ctr_embed_fm2_fwd_sharded_ids32: null shard_ptrs/field_row_offset/ids");
  CTR_REQUIRE(tile || fm2, "ctr_embed_fm2_fwd_sharded_ids32: both outputs are NULL");
  PeerTables peers;
  rc = fill_peers("ctr_embed_fm2_fwd_sharded_ids32", peers, shard_ptrs, G);
  if (rc) return rc;
  CTR_REQUIRE(aligned16(tile), "ctr_embed_fm2_fwd_sharded_ids32: tile must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  return dispatch_fwd(nullptr, &peers, field_row_offset, reinterpret_cast<const int*>(ids), B, F, D, tile, fm2, ids64_out,
                      as_stream(stream));
}

extern "C" int ctr_embed_fm2_bwd(const float* tile, const float* d_tile, const float* d_fm2, int64_t B, int64_t F,
                                 int64_t D, float* row_grads, void* stream) {
  int rc = check_bfd("ctr_embed_fm2_bwd", B, F, D);
  if (rc) return rc;
  CTR_REQUIRE(tile && row_grads, "ctr_embed_fm2_bwd: null tile/row_grads");
  CTR_REQUIRE(aligned16(tile) && aligned16(d_tile) && aligned16(row_grads),
              "ctr_embed_fm2_bwd: tile, d_tile and row_grads must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  return launch_bwd<FM2_PLAIN>("ctr_embed_fm2_bwd", tile, d_tile, d_fm2, nullptr, B, F, D, row_grads, nullptr, as_stream(stream));
}

extern "C" int ctr_embed_scatter_add(float* grad_table, const int64_t* field_row_offset, const int64_t* ids,
                                     const float* row_grads, int64_t B, int64_t F, int64_t D, void* stream) {
  int rc = check_bfd("ctr_embed_scatter_add", B, F, D);
  if (rc) return rc;
  CTR_REQUIRE(grad_table && field_row_offset && ids && row_grads, "ctr_embed_scatter_add: null argument");
  CTR_REQUIRE(aligned16(grad_table) && aligned16(row_grads), "ctr_embed_scatter_add: buffers must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  const long long total = (long long)B * F * (D / 4);
  const int grid = capped_grid((total + 255) / 256, (long long)sm_count() * 16);
  return with_lpr(D, [&](auto LPR) {
    return launch("ctr_embed_scatter_add", embed_scatter_add_kernel<LPR>, grid, 256, 0, st, reinterpret_cast<float4*>(grad_table),
                  reinterpret_cast<const long long*>(field_row_offset), reinterpret_cast<const long long*>(ids),
                  reinterpret_cast<const float4*>(row_grads), (int)B, (int)F);
  });
}

static int bag_group(int64_t D) {
  int G = 1;
  while (G < D && G < 32) G <<= 1;
  return G;
}

extern "C" int ctr_bag_lookup_fwd(const float* table, int64_t V, int64_t D, const int64_t* ids,
                                  const int64_t* offsets, int64_t B, float* out, int64_t out_stride, void* stream) {
  CTR_REQUIRE(table && offsets && out, "ctr_bag_lookup_fwd: null argument");
  CTR_REQUIRE(B >= 0 && V >= 0 && D >= 1 && out_stride >= D, "ctr_bag_lookup_fwd: bad sizes");
  CTR_UNSUPPORTED(D > 256, "ctr_bag_lookup_fwd: D=%lld > 256", (long long)D);
  if (B == 0) return CTR_OK;
  const int G = bag_group(D);
  return launch("ctr_bag_lookup_fwd", bag_lookup_fwd_kernel, capped_grid(((long long)B * G + 255) / 256, (long long)sm_count() * 16),
                256, 0, as_stream(stream), table, V, (int)D, reinterpret_cast<const long long*>(ids),
                reinterpret_cast<const long long*>(offsets), (int)B, out, out_stride, G);
}

extern "C" int ctr_bag_lookup_bwd(const float* d_out, int64_t out_stride, int64_t V, int64_t D, const int64_t* ids,
                                  const int64_t* offsets, int64_t B, float* row_grads, void* stream) {
  CTR_REQUIRE(d_out && offsets, "ctr_bag_lookup_bwd: null argument");
  CTR_REQUIRE(B >= 0 && V >= 0 && D >= 1 && out_stride >= D, "ctr_bag_lookup_bwd: bad sizes");
  CTR_UNSUPPORTED(D > 256, "ctr_bag_lookup_bwd: D=%lld > 256", (long long)D);
  if (B == 0) return CTR_OK;
  const int G = bag_group(D);
  return launch("ctr_bag_lookup_bwd", bag_lookup_bwd_kernel, capped_grid(((long long)B * G + 255) / 256, (long long)sm_count() * 16),
                256, 0, as_stream(stream), d_out, out_stride, V, (int)D, reinterpret_cast<const long long*>(ids),
                reinterpret_cast<const long long*>(offsets), (int)B, row_grads, G);
}

extern "C" int ctr_first_order_fwd(const float* w, const int64_t* field_row_offset, const int64_t* ids, int64_t B,
                                   int64_t F, float bias, float* out, void* stream) {
  CTR_REQUIRE(w && field_row_offset && ids && out, "ctr_first_order_fwd: null argument");
  CTR_REQUIRE(B >= 0 && F >= 1 && B <= 0x7fffffffLL / 8 && F <= 65536, "ctr_first_order_fwd: bad sizes");
  if (B == 0) return CTR_OK;
  return launch("ctr_first_order_fwd", first_order_fwd_kernel, capped_grid((B + 7) / 8, (long long)sm_count() * 8), 256, 0,
                as_stream(stream), w, reinterpret_cast<const long long*>(field_row_offset), reinterpret_cast<const long long*>(ids),
                (int)B, (int)F, bias, out);
}

// ---- NFM bi-interaction pooling (SURVEY 8f.4): the same gather, (B, D) output instead of the FM2 scalar ------------------
extern "C" int ctr_embed_bi_fwd(const float* table, const int64_t* field_row_offset, const int64_t* ids, int64_t B, int64_t F,
                                int64_t D, float* tile, float* bi, void* stream) {
  int rc = check_bfd("ctr_embed_bi_fwd", B, F, D);
  if (rc) return rc;
  CTR_REQUIRE(table && field_row_offset && ids && bi, "ctr_embed_bi_fwd: null table/field_row_offset/ids/bi");
  CTR_REQUIRE(aligned16(table) && aligned16(tile) && aligned16(bi), "ctr_embed_bi_fwd: table, tile and bi must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  return with_lpr(D, [&](auto LPR) { return launch_fwd_bi<LPR>(table, field_row_offset, ids, B, F, tile, bi, st); });
}

extern "C" int ctr_embed_bi_bwd(const float* tile, const float* d_tile, const float* d_bi, int64_t B, int64_t F, int64_t D,
                                float* row_grads, void* stream) {
  int rc = check_bfd("ctr_embed_bi_bwd", B, F, D);
  if (rc) return rc;
  CTR_REQUIRE(tile && d_bi && row_grads, "ctr_embed_bi_bwd: null tile/d_bi/row_grads");
  CTR_REQUIRE(aligned16(tile) && aligned16(d_tile) && aligned16(d_bi) && aligned16(row_grads),
              "ctr_embed_bi_bwd: tile, d_tile, d_bi and row_grads must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  return launch_bwd<FM2_BI>("ctr_embed_fm2_bwd", tile, d_tile, d_bi, nullptr, B, F, D, row_grads, nullptr, as_stream(stream));
}

// ---- lookup + FM2 + fused dense(1) head over the flattened tile (e2e form: the consumer does not re-stream the tile) ------
template <int LPR, typename IdT>
static int launch_fwd_lin(const float* table, const PeerTables* peers, const int64_t* off, const IdT* ids, int64_t B, int64_t F,
                          float* tile, float* fm2, int64_t* ids64_out, const float* wlin, float* lin, cudaStream_t st) {
  auto go = [&](auto k, const float4* tb, const PeerTables& pt) {
    return launch_resident("ctr_embed_fm2_lin_fwd", k, (B + 7) / 8, 256, 0, st, tb, pt, reinterpret_cast<const long long*>(off),
                           ids, (int)B, (int)F, reinterpret_cast<float4*>(tile), fm2, reinterpret_cast<long long*>(ids64_out),
                           reinterpret_cast<const float4*>(wlin), lin);
  };
  if (peers != nullptr) return go(embed_fm2_fwd_kernel<LPR, true, 1, false, IdT, true>, nullptr, *peers);
  // 3 CTAs/SM (85 registers): at the 64 registers of the plain gather this variant spills 88 bytes in its inner loop
  return go(embed_fm2_fwd_kernel<LPR, false, 3, false, IdT, true>, reinterpret_cast<const float4*>(table), PeerTables{});
}

template <typename IdT>
static int dispatch_fwd_lin(const float* table, const PeerTables* peers, const int64_t* off, const IdT* ids, int64_t B, int64_t F,
                            int64_t D, float* tile, float* fm2, int64_t* ids64_out, const float* wlin, float* lin, cudaStream_t st) {
  return with_lpr(D, [&](auto LPR) { return launch_fwd_lin<LPR>(table, peers, off, ids, B, F, tile, fm2, ids64_out, wlin, lin, st); });
}

extern "C" int ctr_embed_fm2_lin_fwd(const float* table, const int64_t* field_row_offset, const void* ids, int ids_are_int32,
                                     int64_t B, int64_t F, int64_t D, const float* wlin, float* tile, float* fm2, float* lin,
                                     int64_t* ids64_out, void* stream) {
  int rc = check_bfd("ctr_embed_fm2_lin_fwd", B, F, D);
  if (rc) return rc;
  CTR_REQUIRE(table && field_row_offset && ids && wlin && lin, "ctr_embed_fm2_lin_fwd: null table/field_row_offset/ids/wlin/lin");
  CTR_REQUIRE(aligned16(table) && aligned16(tile) && aligned16(wlin), "ctr_embed_fm2_lin_fwd: table, tile and wlin must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  if (ids_are_int32)
    return dispatch_fwd_lin(table, nullptr, field_row_offset, reinterpret_cast<const int*>(ids), B, F, D, tile, fm2, ids64_out, wlin, lin, st);
  return dispatch_fwd_lin(table, nullptr, field_row_offset, reinterpret_cast<const long long*>(ids), B, F, D, tile, fm2, nullptr, wlin, lin, st);
}

extern "C" int ctr_embed_fm2_lin_fwd_sharded(const float* const* shard_ptrs, int64_t G, const int64_t* field_row_offset,
                                             const void* ids, int ids_are_int32, int64_t B, int64_t F, int64_t D, const float* wlin,
                                             float* tile, float* fm2, float* lin, int64_t* ids64_out, void* stream) {
  int rc = check_bfd("ctr_embed_fm2_lin_fwd_sharded", B, F, D);
  if (rc) return rc;
  CTR_REQUIRE(shard_ptrs && field_row_offset && ids && wlin && lin, "ctr_embed_fm2_lin_fwd_sharded: null argument");
  PeerTables peers;
  rc = fill_peers("ctr_embed_fm2_lin_fwd_sharded", peers, shard_ptrs, G);
  if (rc) return rc;
  CTR_REQUIRE(aligned16(tile) && aligned16(wlin), "ctr_embed_fm2_lin_fwd_sharded: tile and wlin must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  if (ids_are_int32)
    return dispatch_fwd_lin(nullptr, &peers, field_row_offset, reinterpret_cast<const int*>(ids), B, F, D, tile, fm2, ids64_out, wlin, lin, st);
  return dispatch_fwd_lin(nullptr, &peers, field_row_offset, reinterpret_cast<const long long*>(ids), B, F, D, tile, fm2, nullptr, wlin, lin, st);
}

extern "C" int ctr_embed_fm2_lin_bwd(const float* tile, const float* wlin, const float* d_fm2, const float* d_lin, int64_t B,
                                     int64_t F, int64_t D, float* row_grads, float* d_wlin, void* stream) {
  int rc = check_bfd("ctr_embed_fm2_lin_bwd", B, F, D);
  if (rc) return rc;
  CTR_REQUIRE(tile && wlin && row_grads && d_wlin, "ctr_embed_fm2_lin_bwd: null tile/wlin/row_grads/d_wlin");
  CTR_REQUIRE(aligned16(tile) && aligned16(wlin) && aligned16(row_grads) && aligned16(d_wlin),
              "ctr_embed_fm2_lin_bwd: buffers must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(d_wlin, 0, sizeof(float) * F * D, st));
  if (B == 0) return CTR_OK;
  return launch_bwd<FM2_LIN>("ctr_embed_fm2_lin_bwd", tile, wlin, d_fm2, d_lin, B, F, D, row_grads, d_wlin, st);
}

// ---- sequence lookup: (B, T) ids into ONE table -> (B, T, D), zero rows for id -1 / out of range (the zero padding of
// tf.contrib.feature_column.sequence_input_layer, DIN/din.py:209-214) -------------------------------------------------------
template <int LPR>
static int launch_seq(const float* table, const int64_t* range2, const int64_t* ids, int64_t B, int64_t T, float* out, cudaStream_t st) {
  return launch_resident("ctr_embed_seq_fwd", embed_fm2_fwd_kernel<LPR, false, 4, false, long long, false, true>, (B + 7) / 8, 256,
                         0, st, reinterpret_cast<const float4*>(table), PeerTables{}, reinterpret_cast<const long long*>(range2),
                         reinterpret_cast<const long long*>(ids), (int)B, (int)T, reinterpret_cast<float4*>(out), nullptr, nullptr,
                         nullptr, nullptr);
}

extern "C" int ctr_embed_seq_fwd(const float* table, const int64_t* row_range, const int64_t* ids, int64_t B, int64_t T, int64_t D,
                                 float* out, void* stream) {
  int rc = check_bfd("ctr_embed_seq_fwd", B, T > 0 ? T : 1, D);
  if (rc) return rc;
  CTR_REQUIRE(table && row_range && out && (ids || B * T == 0), "ctr_embed_seq_fwd: null argument");
  CTR_REQUIRE(aligned16(table) && aligned16(out), "ctr_embed_seq_fwd: table and out must be 16-byte aligned");
  if (B == 0 || T == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  return with_lpr(D, [&](auto LPR) { return launch_seq<LPR>(table, row_range, ids, B, T, out, st); });
}

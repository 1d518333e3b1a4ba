// Row (e) of SURVEY.md section 8: row-sharded embedding tables across the GPUs of one NVSwitch box.
//
// The reference has no multi-device code (the only trace is a commented parameter-server block,
// WideAndDeep/wide_and_deep.py:41-51).  Semantics kept: the table gradient is the IndexedSlices pair (row, value) and it
// has to reach the row's owner before the optimizer can apply it.
//
// Layout: global row gr (= field_row_offset[f] + id) is owned by rank gr % G and stored at local row gr / G.
//   forward : ctr_embed_fm2_fwd_sharded (embed_fm2.cu) PULLS rows from the owners' shards through NVLink peer mappings
//             inside the gather kernel itself -- no id exchange, no return all-to-all.
//   plan    : ctr_sharded_plan (one pass over the ids, independent of the forward): every valid (b,f) gets a slot in its
//             owner's receive queue -- CTA-level counting in shared memory, ONE global atomic per CTA chunk and owner -- and
//             the queue's row indices are staged per owner in shared memory and leave as contiguous runs (8-byte scattered
//             peer stores would cost a link packet each).  The last CTA publishes the per-owner counts.
//   backward: ctr_embed_fm2_bwd_push computes the IndexedSlices values d_tile + g*(S - e) in registers and stores each row
//             STRAIGHT into its owner's queue with 128-bit peer stores: the all-to-all(v) of the gradients is fused into the
//             backward kernel and row_grads never touches local HBM.  ctr_sharded_grad_push is the same exchange for row
//             gradients that already exist (any other interaction layer upstream).
//   After a stream sync + cross-rank barrier the owner consumes (rows, values, count) with ctr_adam_rows_dedup or
//   ctr_rows_scatter_add.
// Measured link ceilings for this access pattern (tools/peerbench.cu, all ranks active at once, 128-byte rows): pull
// 650 GB/s with L1-allocating loads (622 with .nc.L1::no_allocate), push 680-690 GB/s with plain 128-bit stores, per
// direction per rank; random rows == sequential rows, bulk-async (TMA) copies == LDG/STG, 8 GB == 32 GB shards.
#include "lookup_bwd.cuh"

namespace ctr {

struct PeerQueues {
  float4* vals[8];          // owner d: (G_src, capacity, D) fp32
  long long* rows[8];       // owner d: (G_src, capacity) int64 local rows
  long long* counts[8];     // owner d: (G_src,) int64 filled slots per source (published by the plan kernel)
  int G, logG, my_rank;
  long long capacity;
};

constexpr int PLAN_THREADS = 256;
constexpr int PLAN_IPT = 5;                          // ids per thread and chunk
constexpr int PLAN_CHUNK = PLAN_THREADS * PLAN_IPT;  // 1280 ids = 32 samples at F = 40
constexpr int PLAN_SLOT_BITS = 28;                   // plan word = owner << 28 | slot ; -1 = invalid id / dropped
constexpr int PLAN_SLOT_MASK = (1 << PLAN_SLOT_BITS) - 1;

__device__ __forceinline__ long long plan_load_id(const long long* p) { return ldg_stream_i64(p); }
__device__ __forceinline__ long long plan_load_id(const int* p) { return (long long)__ldg(p); }

template <typename IdT>
__global__ void __launch_bounds__(PLAN_THREADS)
sharded_plan_kernel(const long long* __restrict__ row_off, const IdT* __restrict__ ids, long long n, int F,
                    const PeerQueues q, unsigned long long* __restrict__ counters, int* __restrict__ overflow,
                    int* __restrict__ plan) {
  __shared__ unsigned int s_cnt[8], s_off[9];
  __shared__ unsigned long long s_base[8];
  __shared__ long long s_rows[PLAN_CHUNK];
  __shared__ int s_last;
  const int tid = threadIdx.x, G = q.G;
  const long long nchunks = (n + PLAN_CHUNK - 1) / PLAN_CHUNK;
  for (long long ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
    if (tid < 8) s_cnt[tid] = 0;
    __syncthreads();
    int owner[PLAN_IPT];
    unsigned int pos[PLAN_IPT];
    long long lrow[PLAN_IPT];
#pragma unroll
    for (int k = 0; k < PLAN_IPT; ++k) {
      const long long e = ch * PLAN_CHUNK + k * PLAN_THREADS + tid;
      owner[k] = -1; pos[k] = 0; lrow[k] = 0;
      if (e < n) {
        const int f = (int)(e % F);
        const long long id = plan_load_id(ids + e);
        const long long lo = __ldg(row_off + f), hi = __ldg(row_off + f + 1);
        if (id >= 0 && id < hi - lo) {
          owner[k] = (int)((lo + id) & (G - 1));
          lrow[k] = (lo + id) >> q.logG;
          pos[k] = atomicAdd(&s_cnt[owner[k]], 1u);
        }
      }
    }
    __syncthreads();
    if (tid < G) s_base[tid] = atomicAdd(&counters[tid], (unsigned long long)s_cnt[tid]);
    if (tid == 32) {
      unsigned int acc = 0;
      for (int d = 0; d < 8; ++d) { s_off[d] = acc; acc += d < G ? s_cnt[d] : 0u; }
      s_off[8] = acc;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < PLAN_IPT; ++k) {
      const long long e = ch * PLAN_CHUNK + k * PLAN_THREADS + tid;
      if (e < n) {
        int word = -1;
        if (owner[k] >= 0) {
          const unsigned long long slot = s_base[owner[k]] + pos[k];
          s_rows[s_off[owner[k]] + pos[k]] = lrow[k];
          if (slot < (unsigned long long)q.capacity) word = (owner[k] << PLAN_SLOT_BITS) | (int)slot;
          else atomicOr(overflow, 1);
        }
        plan[e] = word;
      }
    }
    __syncthreads();
    // the chunk's row indices leave as one contiguous run per owner
    const unsigned int total = s_off[8];
    for (unsigned int j = tid; j < total; j += PLAN_THREADS) {
      int d = 0;
#pragma unroll
      for (int t = 1; t < 8; ++t) d += (t < G && j >= s_off[t]) ? 1 : 0;
      const unsigned long long slot = s_base[d] + (j - s_off[d]);
      if (slot < (unsigned long long)q.capacity) q.rows[d][(size_t)q.my_rank * q.capacity + slot] = s_rows[j];
    }
    __syncthreads();
  }
  // the last CTA to finish publishes how many entries this rank queued at every owner (clamped to the capacity)
  __threadfence();
  if (tid == 0) s_last = atomicAdd(&counters[8], 1ull) == (unsigned long long)gridDim.x - 1;
  __syncthreads();
  if (s_last && tid < G) {
    unsigned long long c = atomicAdd(&counters[tid], 0ull);
    if (c > (unsigned long long)q.capacity) c = (unsigned long long)q.capacity;
    if (q.counts[tid] != nullptr) q.counts[tid][q.my_rank] = (long long)c;
  }
}

__device__ __forceinline__ void stg_f4(float4* p, const float4& v) {
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4* queue_slot(const PeerQueues& q, size_t qbase, int word, int lpr, int c) {
  return q.vals[word >> PLAN_SLOT_BITS] + (qbase + (size_t)(word & PLAN_SLOT_MASK)) * lpr + c;
}

// Sink of the push backward: every finished 128-bit piece goes to owner.vals[(my_rank*capacity + slot)*LPR + c] (and to
// row_grads when given).  PREFETCH: the plan words are loaded with the d_tile rows, before the S reduction, and held in
// registers; otherwise each is loaded at use.  The LIN form loads at use: with the d_wlin accumulator in registers,
// holding the plan words as well spills under its 2-CTA bound at HOLD = 12.
template <int LPR, int HOLD, bool PREFETCH>
struct QueueSink {
  const PeerQueues& q;
  size_t qbase;
  const int* __restrict__ p_row;
  float4* __restrict__ o_row;
  int pw[PREFETCH ? HOLD : 1];
  __device__ __forceinline__ void fetch(int k, int j) {
    if (PREFETCH) pw[k] = __ldg(p_row + j / LPR);
  }
  __device__ __forceinline__ void operator()(int k, int j, const float4& r) {
    if (o_row != nullptr) stg_stream_f4(o_row + j, r);
    const int w = PREFETCH ? pw[k] : __ldg(p_row + j / LPR);
    if (w >= 0) stg_f4(queue_slot(q, qbase, w, LPR, j % LPR), r);
  }
};

// Lookup backward fused with the gradient exchange: the per-sample body of lookup_bwd.cuh with the queue store as sink.
// LIN (HOLD > 0 only): the backward of the fused dense(1) head (ctr_embed_fm2_lin_fwd), as in embed_fm2_bwd_kernel:
// `d_tile` carries wlin (F*D) and d_wlin = sum_b d_lin[b]*e[b] is accumulated (LinHead).
template <int LPR, int HOLD, bool LIN = false>
__global__ void __launch_bounds__(256, LIN ? 2 : 1)
embed_fm2_bwd_push_kernel(const float4* __restrict__ tile, const float4* __restrict__ d_tile, const float* __restrict__ d_fm2,
                          const int* __restrict__ plan, int B, int F, const PeerQueues q, float4* __restrict__ row_grads,
                          const float* __restrict__ d_lin, float4* __restrict__ d_wlin) {
  extern __shared__ float4 s_lin[];
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int n4 = F * LPR;
  const size_t qbase = (size_t)q.my_rank * q.capacity;
  LinHead<LIN ? HOLD : 1> lin;
  if (LIN) lin.stage(s_lin, d_tile, n4);
  for (int b = warp0; b < B; b += nwarps) {
    const float4* e_row = tile + (size_t)b * n4;
    RowGrad rows{(d_tile && !LIN) ? d_tile + (size_t)b * n4 : nullptr};
    QueueSink<LPR, HOLD, (HOLD > 0 && !LIN)> sink{q, qbase, plan + (size_t)b * F, row_grads ? row_grads + (size_t)b * n4 : nullptr};
    const float g = d_fm2 ? __ldg(d_fm2 + b) : 0.f;
    const float4 g4 = make_float4(g, g, g, g);
    if constexpr (LIN) {
      lin.gl = d_lin ? __ldg(d_lin + b) : 0.f;
      lookup_bwd_sample<LPR, HOLD>(e_row, n4, lane, g4, lin, sink);
    } else {
      lookup_bwd_sample<LPR, HOLD>(e_row, n4, lane, g4, rows, sink);
    }
  }
  if (LIN) lin.flush(d_wlin, lane);
}

// The exchange alone: row_grads (B,F,D) already exist; every planned row is copied into its owner's queue.
template <int LPR>
__global__ void __launch_bounds__(256)
sharded_push_rows_kernel(const float4* __restrict__ row_grads, const int* __restrict__ plan, long long n_rows, const PeerQueues q) {
  const size_t total = (size_t)n_rows * LPR;
  const size_t qbase = (size_t)q.my_rank * q.capacity;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int pw = __ldg(plan + t / LPR);
    if (pw >= 0) stg_f4(queue_slot(q, qbase, pw, LPR, (int)(t % LPR)), ldg_stream_f4(row_grads + t));
  }
}

// dst[rows[i], :] += vals[i, :] for i < min(*count, max_n); rows outside [0, V) are ignored.
template <int LPR>
__global__ void __launch_bounds__(256)
rows_scatter_add_kernel(float4* __restrict__ dst, long long V, const long long* __restrict__ rows,
                        const float4* __restrict__ vals, const long long* __restrict__ count, long long max_n) {
  long long n = count ? *count : max_n;
  if (n > max_n) n = max_n;
  const size_t total = (size_t)n * LPR;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const long long row = __ldg(rows + t / LPR);
    if (row >= 0 && row < V) atomicAdd(dst + (size_t)row * LPR + t % LPR, ldg_stream_f4(vals + t));
  }
}

static int check_g(const char* fn, int64_t G, int64_t rank) {
  CTR_REQUIRE(G >= 1 && G <= 8 && (G & (G - 1)) == 0, "%s: G=%lld must be a power of two <= 8", fn, (long long)G);
  CTR_REQUIRE(rank >= 0 && rank < G, "%s: rank %lld out of range", fn, (long long)rank);
  return CTR_OK;
}

static int fill_queues(const char* fn, PeerQueues& q, int64_t G, int64_t my_rank, float* const* recv_vals,
                       int64_t* const* recv_rows, int64_t* const* recv_counts, int64_t capacity) {
  int rc = check_g(fn, G, my_rank);
  if (rc) return rc;
  CTR_REQUIRE(capacity >= 0 && capacity <= PLAN_SLOT_MASK, "%s: capacity %lld must be in [0, 2^28)", fn, (long long)capacity);
  q = PeerQueues{};
  q.G = (int)G;
  while ((1 << q.logG) < G) ++q.logG;
  q.my_rank = (int)my_rank;
  q.capacity = capacity;
  for (int r = 0; r < G; ++r) {
    if (recv_vals) {
      CTR_REQUIRE(recv_vals[r] && aligned16(recv_vals[r]), "%s: value queue %d null/unaligned", fn, r);
      q.vals[r] = reinterpret_cast<float4*>(recv_vals[r]);
    }
    if (recv_rows) {
      CTR_REQUIRE(recv_rows[r] != nullptr, "%s: row queue %d is null", fn, r);
      q.rows[r] = reinterpret_cast<long long*>(recv_rows[r]);
    }
    if (recv_counts) q.counts[r] = reinterpret_cast<long long*>(recv_counts[r]);
  }
  return CTR_OK;
}

}  // namespace ctr

using namespace ctr;

extern "C" int ctr_sharded_plan(const int64_t* field_row_offset, const void* ids, int ids_are_int32, int64_t B, int64_t F, int64_t G,
                                int64_t my_rank, int64_t* const* recv_rows, int64_t* const* recv_counts, int64_t capacity,
                                int64_t* counters, int* overflow, int32_t* plan, void* stream) {
  PeerQueues q;
  int rc = fill_queues("ctr_sharded_plan", q, G, my_rank, nullptr, recv_rows, recv_counts, capacity);
  if (rc) return rc;
  CTR_REQUIRE(field_row_offset && ids && recv_rows && counters && overflow && plan, "ctr_sharded_plan: null argument");
  CTR_REQUIRE(B >= 0 && F >= 1 && B * F <= PLAN_SLOT_MASK, "ctr_sharded_plan: bad sizes (B*F must be < 2^28)");
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(counters, 0, sizeof(int64_t) * 9, st));
  CTR_CUDA(cudaMemsetAsync(overflow, 0, sizeof(int), st));
  const long long n = (long long)B * F;
  const long long chunks = (n + PLAN_CHUNK - 1) / PLAN_CHUNK;
  // B == 0 still runs one CTA: it publishes the zero counts
  const int grid = capped_grid(chunks < 1 ? 1 : chunks, (long long)sm_count() * 4);
  auto go = [&](auto k, auto typed_ids) {
    return launch("ctr_sharded_plan", k, grid, PLAN_THREADS, 0, st, reinterpret_cast<const long long*>(field_row_offset), typed_ids, n,
                  (int)F, q, reinterpret_cast<unsigned long long*>(counters), overflow, plan);
  };
  return ids_are_int32 ? go(sharded_plan_kernel<int>, static_cast<const int*>(ids))
                       : go(sharded_plan_kernel<long long>, static_cast<const long long*>(ids));
}

extern "C" int ctr_embed_fm2_bwd_push(const float* tile, const float* d_tile, const float* d_fm2, const int32_t* plan, int64_t B,
                                      int64_t F, int64_t D, int64_t G, int64_t my_rank, float* const* recv_vals,
                                      int64_t capacity, float* row_grads, void* stream) {
  PeerQueues q;
  int rc = fill_queues("ctr_embed_fm2_bwd_push", q, G, my_rank, recv_vals, nullptr, nullptr, capacity);
  if (rc) return rc;
  CTR_REQUIRE(tile && plan && recv_vals, "ctr_embed_fm2_bwd_push: null tile/plan/recv_vals");
  CTR_REQUIRE(B >= 0 && F >= 1 && B <= 0x7fffffffLL / 8 && F <= 65536, "ctr_embed_fm2_bwd_push: bad sizes");
  CTR_UNSUPPORTED(D % 4 != 0 || D > 128 || (D & (D - 1)) != 0, "ctr_embed_fm2_bwd_push: D=%lld unsupported", (long long)D);
  CTR_REQUIRE(aligned16(tile) && aligned16(d_tile) && aligned16(row_grads),
              "ctr_embed_fm2_bwd_push: tile, d_tile and row_grads must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  return with_lpr(D, [&](auto LPR) {
    return with_hold<true>(F, LPR, [&](auto HOLD) {
      return launch_resident("ctr_embed_fm2_bwd_push", embed_fm2_bwd_push_kernel<LPR, HOLD, false>, (B + 7) / 8, 256, 0,
                             as_stream(stream), reinterpret_cast<const float4*>(tile), reinterpret_cast<const float4*>(d_tile), d_fm2,
                             plan, (int)B, (int)F, q, reinterpret_cast<float4*>(row_grads), nullptr, nullptr);
    });
  });
}

extern "C" int ctr_embed_fm2_lin_bwd_push(const float* tile, const float* wlin, const float* d_fm2, const float* d_lin,
                                          const int32_t* plan, int64_t B, int64_t F, int64_t D, int64_t G, int64_t my_rank,
                                          float* const* recv_vals, int64_t capacity, float* row_grads, float* d_wlin,
                                          void* stream) {
  PeerQueues q;
  int rc = fill_queues("ctr_embed_fm2_lin_bwd_push", q, G, my_rank, recv_vals, nullptr, nullptr, capacity);
  if (rc) return rc;
  CTR_REQUIRE(tile && wlin && plan && recv_vals && d_wlin, "ctr_embed_fm2_lin_bwd_push: null tile/wlin/plan/recv_vals/d_wlin");
  CTR_REQUIRE(B >= 0 && F >= 1 && B <= 0x7fffffffLL / 8 && F <= 65536, "ctr_embed_fm2_lin_bwd_push: bad sizes");
  CTR_UNSUPPORTED(D % 4 != 0 || D > 128 || (D & (D - 1)) != 0, "ctr_embed_fm2_lin_bwd_push: D=%lld unsupported", (long long)D);
  CTR_REQUIRE(aligned16(tile) && aligned16(wlin) && aligned16(row_grads) && aligned16(d_wlin),
              "ctr_embed_fm2_lin_bwd_push: tile, wlin, row_grads and d_wlin must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  CTR_CUDA(cudaMemsetAsync(d_wlin, 0, sizeof(float) * F * D, st));
  if (B == 0) return CTR_OK;
  return with_lpr(D, [&](auto LPR) {
    return with_hold<false>(F, LPR, [&](auto HOLD) {
      return launch_resident("ctr_embed_fm2_lin_bwd_push", embed_fm2_bwd_push_kernel<LPR, HOLD, true>, (B + 7) / 8, 256,
                             sizeof(float4) * 2 * (size_t)F * LPR, st, reinterpret_cast<const float4*>(tile),
                             reinterpret_cast<const float4*>(wlin), d_fm2, plan, (int)B, (int)F, q,
                             reinterpret_cast<float4*>(row_grads), d_lin, reinterpret_cast<float4*>(d_wlin));
    }, "ctr_embed_fm2_lin_bwd_push");
  });
}

extern "C" int ctr_sharded_grad_push(const float* row_grads, const int32_t* plan, int64_t B, int64_t F, int64_t D, int64_t G,
                                     int64_t my_rank, float* const* recv_vals, int64_t capacity, void* stream) {
  PeerQueues q;
  int rc = fill_queues("ctr_sharded_grad_push", q, G, my_rank, recv_vals, nullptr, nullptr, capacity);
  if (rc) return rc;
  CTR_REQUIRE(row_grads && plan && recv_vals, "ctr_sharded_grad_push: null argument");
  CTR_REQUIRE(B >= 0 && F >= 1, "ctr_sharded_grad_push: bad sizes");
  CTR_UNSUPPORTED(D % 4 != 0 || D > 128 || (D & (D - 1)) != 0, "ctr_sharded_grad_push: D=%lld unsupported", (long long)D);
  CTR_REQUIRE(aligned16(row_grads), "ctr_sharded_grad_push: row_grads must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  const long long n_rows = (long long)B * F, total = n_rows * (D / 4);
  const int grid = capped_grid((total + 255) / 256, (long long)sm_count() * 8);
  return with_lpr(D, [&](auto LPR) {
    return launch("ctr_sharded_grad_push", sharded_push_rows_kernel<LPR>, grid, 256, 0, st, reinterpret_cast<const float4*>(row_grads),
                  plan, n_rows, q);
  });
}

extern "C" int ctr_rows_scatter_add(float* dst, int64_t V, int64_t D, const int64_t* rows, const float* vals,
                                    const int64_t* count, int64_t max_n, void* stream) {
  CTR_REQUIRE(dst && rows && vals, "ctr_rows_scatter_add: null argument");
  CTR_REQUIRE(V >= 0 && max_n >= 0, "ctr_rows_scatter_add: bad sizes");
  CTR_UNSUPPORTED(D % 4 != 0 || D > 128 || (D & (D - 1)) != 0, "ctr_rows_scatter_add: D=%lld unsupported", (long long)D);
  CTR_REQUIRE(aligned16(dst) && aligned16(vals), "ctr_rows_scatter_add: buffers must be 16-byte aligned");
  if (max_n == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  const long long total = (long long)max_n * (D / 4);
  const int grid = capped_grid((total + 255) / 256, (long long)sm_count() * 16);
  return with_lpr(D, [&](auto LPR) {
    return launch("ctr_rows_scatter_add", rows_scatter_add_kernel<LPR>, grid, 256, 0, st, reinterpret_cast<float4*>(dst), V,
                  reinterpret_cast<const long long*>(rows), reinterpret_cast<const float4*>(vals),
                  reinterpret_cast<const long long*>(count), max_n);
  });
}

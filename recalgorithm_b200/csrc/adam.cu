// SURVEY.md 8f.3 -- the step right after the hot path: applying the IndexedSlices gradient to the embedding table.
//
// Reference: tf.train.AdamOptimizer(lr, 0.9, 0.999, 1e-8) on every variable (DeepFM/deepfm.py:246-250); for a table its
// gradient is IndexedSlices and TF's _apply_sparse [TF-internal, SURVEY A.8] does
//     g  = unsorted_segment_sum(values, indices)                  (duplicates summed FIRST; g*g is on the sum)
//     m <- b1*m (DENSE)   ; m[idx] += (1-b1)*g        v <- b2*v (DENSE) ; v[idx] += (1-b2)*g*g
//     var <- var - lr_t * m / (sqrt(v) + eps)   (DENSE),    lr_t = lr*sqrt(1-b2^t)/(1-b1^t)
// i.e. plain Adam on the densified gradient: every row of the table moves every step.  DIEN alone uses LazyAdam
// (DIEN/dien.py:328): only the referenced rows are touched.
//
// H100 mapping (pure HBM streaming, no tensor cores): the caller de-duplicates rows and sums their values (one
// ctr_rows_scatter_add into a compact buffer); then
//   ctr_adam_rows        updates m, v, var of the U referenced rows and marks them in a bitmap   (both variants)
//   ctr_adam_dense_rest  streams over ALL other rows with g = 0: m*=b1, v*=b2, var -= lr_t*m/(sqrt(v)+eps)   (TF variant only)
// so the faithful variant costs 6 table-sized streams per step (77 GB at config 5 -> ~12 ms at HBM peak, 40x the hot
// path itself) and the lazy variant a few hundred MB.
#include "ctr_common.cuh"

namespace ctr {

template <int LPR>
__global__ void __launch_bounds__(256)
adam_rows_kernel(float4* __restrict__ var, float4* __restrict__ m, float4* __restrict__ v, int SS, long long V,
                 const long long* __restrict__ rows, const float4* __restrict__ grads, const long long* __restrict__ count,
                 long long max_n, float lr_t, float b1, float b2, float eps, unsigned int* __restrict__ touched) {
  long long n = count ? *count : max_n;
  if (n > max_n) n = max_n;
  const size_t total = (size_t)n * LPR;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const long long row = __ldg(rows + t / LPR);
    if (row < 0 || row >= V) continue;
    const size_t off = (size_t)row * LPR + t % LPR, so = (size_t)row * SS + t % LPR;
    const float4 g = ldg_stream_f4(grads + t);
    float4 mm = m[so], vv = v[so], w = var[off];
    mm.x = b1 * mm.x + (1.f - b1) * g.x; mm.y = b1 * mm.y + (1.f - b1) * g.y;
    mm.z = b1 * mm.z + (1.f - b1) * g.z; mm.w = b1 * mm.w + (1.f - b1) * g.w;
    vv.x = b2 * vv.x + (1.f - b2) * g.x * g.x; vv.y = b2 * vv.y + (1.f - b2) * g.y * g.y;
    vv.z = b2 * vv.z + (1.f - b2) * g.z * g.z; vv.w = b2 * vv.w + (1.f - b2) * g.w * g.w;
    w.x -= lr_t * mm.x / (sqrtf(vv.x) + eps); w.y -= lr_t * mm.y / (sqrtf(vv.y) + eps);
    w.z -= lr_t * mm.z / (sqrtf(vv.z) + eps); w.w -= lr_t * mm.w / (sqrtf(vv.w) + eps);
    m[so] = mm; v[so] = vv; var[off] = w;
    if (touched != nullptr && t % LPR == 0) atomicOr(touched + (row >> 5), 1u << (row & 31));
  }
}

template <int LPR>
__global__ void __launch_bounds__(256)
adam_dense_rest_kernel(float4* __restrict__ var, float4* __restrict__ m, float4* __restrict__ v, int SS, long long V, float lr_t,
                       float b1, float b2, float eps, const unsigned int* __restrict__ touched) {
  const size_t total = (size_t)V * LPR;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const long long row = (long long)(t / LPR);
    if (touched != nullptr && (__ldg(touched + (row >> 5)) >> (row & 31)) & 1u) continue;   // done by adam_rows_kernel
    const size_t so = (size_t)row * SS + t % LPR;
    float4 mm = ldg_stream_f4(m + so), vv = ldg_stream_f4(v + so), w = ldg_stream_f4(var + t);
    mm.x *= b1; mm.y *= b1; mm.z *= b1; mm.w *= b1;
    vv.x *= b2; vv.y *= b2; vv.z *= b2; vv.w *= b2;
    w.x -= lr_t * mm.x / (sqrtf(vv.x) + eps); w.y -= lr_t * mm.y / (sqrtf(vv.y) + eps);
    w.z -= lr_t * mm.z / (sqrtf(vv.z) + eps); w.w -= lr_t * mm.w / (sqrtf(vv.w) + eps);
    stg_stream_f4(m + so, mm); stg_stream_f4(v + so, vv); stg_stream_f4(var + t, w);
  }
}

// ---- fused IndexedSlices step: device-side de-duplication without a sort -------------------------------------------------
// slot_of_row (int32 per table row, -1 when idle) elects, per referenced row, the FIRST-claiming (b,f) entry as the row's
// accumulator:  claim (atomicCAS) -> merge (every other entry of that row adds its gradient into the winner's slot of
// row_grads, 128-bit reductions) -> update (the winner applies Adam with the summed gradient, clears the slot, marks the
// bitmap).  Three launches on one stream, no host round trip; row_grads is consumed (clobbered).
// Where the entries of one step come from: the (B,F) id matrix of an IndexedSlices (row = field offset + local id), or the
// receive queues of a row-sharded table (nseg segments of `cap` (row, value) slots, counts[seg] of them filled).
constexpr int DUP_FLAG = 0x40000000;   // set in slot_of_row[row] when a second entry of the batch meets an already claimed row
struct EntrySrc {
  const long long* ids;      // (B,F) local ids | (nseg, cap) local rows
  const long long* off;      // (F+1,) field row offsets | nullptr
  const long long* counts;   // nullptr | (nseg,)
  long long cap, V;          // segment capacity | rows of the table (range check of the flat form)
  int F;
};
__device__ __forceinline__ long long entry_row(const EntrySrc& s, long long e) {
  if (s.off != nullptr) {
    const int f = (int)(e % s.F);
    const long long id = __ldg(s.ids + e), base = __ldg(s.off + f);
    return (id < 0 || id >= __ldg(s.off + f + 1) - base) ? -1 : base + id;
  }
  if (e % s.cap >= __ldg(s.counts + e / s.cap)) return -1;
  const long long row = __ldg(s.ids + e);
  return (row < 0 || row >= s.V) ? -1 : row;
}

__global__ void __launch_bounds__(256)
adam_claim_kernel(const EntrySrc src, long long n, int* __restrict__ slot) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long row = entry_row(src, e);
    if (row >= 0) atomicCAS(slot + row, -1, (int)e);
  }
}

// claim that also LISTS the losing entries (rows met a second time): the merge then walks that list (a few per cent of the
// entries with uniform ids) instead of re-scanning every entry and its slot
__global__ void __launch_bounds__(256)
adam_claim_list_kernel(const EntrySrc src, long long n, int* __restrict__ slot, int* __restrict__ dup_list, int* __restrict__ n_dup) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long row = entry_row(src, e);
    if (row >= 0 && atomicCAS(slot + row, -1, (int)e) != -1) {
      atomicOr(slot + row, DUP_FLAG);
      dup_list[atomicAdd(n_dup, 1)] = (int)e;
    }
  }
}
template <int LPR>
__global__ void __launch_bounds__(256)
adam_merge_list_kernel(const EntrySrc src, const int* __restrict__ slot, float4* __restrict__ grads, const int* __restrict__ dup_list,
                       const int* __restrict__ n_dup) {
  const size_t total = (size_t)(*n_dup) * LPR;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int e = __ldg(dup_list + t / LPR);
    const long long row = entry_row(src, e);
    const int w = __ldg(slot + row) & ~DUP_FLAG;
    atomicAdd(grads + (size_t)w * LPR + t % LPR, grads[(size_t)e * LPR + t % LPR]);
  }
}

template <int LPR>
__global__ void __launch_bounds__(256)
adam_merge_kernel(const EntrySrc src, long long n, const int* __restrict__ slot, float4* __restrict__ grads) {
  const size_t total = (size_t)n * LPR;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const long long e = (long long)(t / LPR);
    const long long row = entry_row(src, e);
    if (row < 0) continue;
    const int w = __ldg(slot + row);
    if (w != (int)e) atomicAdd(grads + (size_t)w * LPR + t % LPR, grads[t]);
  }
}

template <int LPR>
__global__ void __launch_bounds__(256)
adam_update_kernel(float4* __restrict__ var, float4* __restrict__ m, float4* __restrict__ v, int SS, const EntrySrc src, long long n,
                   int* __restrict__ slot, const float4* __restrict__ grads,
                   float lr_t, float b1, float b2, float eps, unsigned int* __restrict__ touched, long long* __restrict__ n_unique) {
  const size_t total = (size_t)n * LPR;
  int mine = 0;
  // warp-uniform trip count: the lanes of one entry (LPR <= 32, aligned) sit in one warp and all read the slot before
  // lane 0 of the entry clears it
  for (size_t base = ((size_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31)); base < total; base += (size_t)gridDim.x * blockDim.x) {
    const size_t t = base + (threadIdx.x & 31);
    long long row = -1;
    bool win = false;
    if (t < total) {
      const long long e = (long long)(t / LPR);
      row = entry_row(src, e);
      win = row >= 0 && (slot[row] & ~DUP_FLAG) == (int)e;
    }
    __syncwarp();
    if (!win) continue;
    const size_t o = (size_t)row * LPR + t % LPR, so = (size_t)row * SS + t % LPR;
    const float4 g = ldg_stream_f4(grads + t);
    float4 mm = m[so], vv = v[so], w = var[o];
    mm.x = b1 * mm.x + (1.f - b1) * g.x; mm.y = b1 * mm.y + (1.f - b1) * g.y;
    mm.z = b1 * mm.z + (1.f - b1) * g.z; mm.w = b1 * mm.w + (1.f - b1) * g.w;
    vv.x = b2 * vv.x + (1.f - b2) * g.x * g.x; vv.y = b2 * vv.y + (1.f - b2) * g.y * g.y;
    vv.z = b2 * vv.z + (1.f - b2) * g.z * g.z; vv.w = b2 * vv.w + (1.f - b2) * g.w * g.w;
    w.x -= lr_t * mm.x / (sqrtf(vv.x) + eps); w.y -= lr_t * mm.y / (sqrtf(vv.y) + eps);
    w.z -= lr_t * mm.z / (sqrtf(vv.z) + eps); w.w -= lr_t * mm.w / (sqrtf(vv.w) + eps);
    m[so] = mm; v[so] = vv; var[o] = w;
    if (t % LPR == 0) {
      slot[row] = -1;
      if (touched != nullptr) atomicOr(touched + (row >> 5), 1u << (row & 31));
      ++mine;
    }
  }
  if (n_unique != nullptr) {
    mine = __reduce_add_sync(0xffffffffu, mine);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(reinterpret_cast<unsigned long long*>(n_unique), (unsigned long long)mine);
  }
}

// ---- lookup backward FUSED with the sparse Adam step (SURVEY 8f.3: "a fused row-wise update avoids writing row-grads to HBM") ----
// claim (as above, plus a DUP flag when a second entry meets an already claimed row) -> ONE pass that computes the
// IndexedSlices values d_tile + g*(S - e) in registers and, for every row referenced once in the batch (~99 % with uniform
// ids), applies Adam on the spot: row_grads is neither written nor re-read.  Rows referenced more than once park their
// values in `dup_grads` and their entry index in `dup_list`; two list-driven launches (merge into the claiming entry, update)
// finish them with the SUMMED gradient, exactly like the unfused path.
__global__ void __launch_bounds__(256)
adam_claim_dup_kernel(const EntrySrc src, long long n, int* __restrict__ slot) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long row = entry_row(src, e);
    if (row >= 0 && atomicCAS(slot + row, -1, (int)e) != -1) atomicOr(slot + row, DUP_FLAG);
  }
}

__device__ __forceinline__ void adam_apply(float4& w, float4& mm, float4& vv, const float4& g, float lr_t, float b1, float b2, float eps) {
  mm.x = b1 * mm.x + (1.f - b1) * g.x; mm.y = b1 * mm.y + (1.f - b1) * g.y;
  mm.z = b1 * mm.z + (1.f - b1) * g.z; mm.w = b1 * mm.w + (1.f - b1) * g.w;
  vv.x = b2 * vv.x + (1.f - b2) * g.x * g.x; vv.y = b2 * vv.y + (1.f - b2) * g.y * g.y;
  vv.z = b2 * vv.z + (1.f - b2) * g.z * g.z; vv.w = b2 * vv.w + (1.f - b2) * g.w * g.w;
  w.x -= lr_t * mm.x / (sqrtf(vv.x) + eps); w.y -= lr_t * mm.y / (sqrtf(vv.y) + eps);
  w.z -= lr_t * mm.z / (sqrtf(vv.z) + eps); w.w -= lr_t * mm.w / (sqrtf(vv.w) + eps);
}

// warp per sample; HOLD float4 per lane cover the sample's F*LPR chunks (F*D <= HOLD*128 floats); GK chunks are in flight
// together in the update phase (d_tile, m, v, var loads issued before the first use).
template <int LPR, int HOLD>
__global__ void __launch_bounds__(256, 1)
embed_fm2_bwd_adam_kernel(const float4* __restrict__ tile, const float4* __restrict__ d_tile, const float* __restrict__ d_fm2,
                          const long long* __restrict__ row_off, const long long* __restrict__ ids, int B, int F,
                          float4* __restrict__ var, float4* __restrict__ m, float4* __restrict__ v, int SS, int* __restrict__ slot,
                          float4* __restrict__ dup_grads, int* __restrict__ dup_list, int* __restrict__ n_dup,
                          float lr_t, float b1, float b2, float eps, unsigned int* __restrict__ touched,
                          long long* __restrict__ n_unique) {
  constexpr int GK = HOLD < 4 ? HOLD : 4;
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int n4 = F * LPR;
  const int c = lane % LPR;
  int mine = 0;
  for (int b = warp0; b < B; b += nwarps) {
    const float4* e_row = tile + (size_t)b * n4;
    const float4* dt_row = d_tile ? d_tile + (size_t)b * n4 : nullptr;
    const float g = d_fm2 ? __ldg(d_fm2 + b) : 0.f;
    float4 e[HOLD];
    long long row[HOLD];
#pragma unroll
    for (int k = 0; k < HOLD; ++k) {
      const int j = k * 32 + lane;
      e[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      row[k] = -1;
      if (j < n4) {
        e[k] = ldg_stream_f4(e_row + j);
        const int f = j / LPR;
        const long long id = __ldg(ids + (size_t)b * F + f), lo = __ldg(row_off + f);
        if (id >= 0 && id < __ldg(row_off + f + 1) - lo) row[k] = lo + id;
      }
    }
    int s[HOLD];
#pragma unroll
    for (int k = 0; k < HOLD; ++k) s[k] = row[k] >= 0 ? __ldg(slot + row[k]) : -1;   // read-only during this launch for non-dup rows' peers
    float4 S = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < HOLD; ++k) { S.x += e[k].x; S.y += e[k].y; S.z += e[k].z; S.w += e[k].w; }
#pragma unroll
    for (int o = LPR; o < 32; o <<= 1) {
      S.x += __shfl_xor_sync(full, S.x, o); S.y += __shfl_xor_sync(full, S.y, o);
      S.z += __shfl_xor_sync(full, S.z, o); S.w += __shfl_xor_sync(full, S.w, o);
    }
#pragma unroll
    for (int k0 = 0; k0 < HOLD; k0 += GK) {
      float4 dt[GK], mm[GK], vv[GK], ww[GK];
#pragma unroll
      for (int u = 0; u < GK; ++u) {
        const int k = k0 + u, j = k * 32 + lane;
        dt[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < HOLD && j < n4 && dt_row != nullptr) dt[u] = ldg_stream_f4(dt_row + j);
        if (k < HOLD && row[k] >= 0 && !(s[k] & DUP_FLAG)) {
          const size_t o = (size_t)row[k] * LPR + c, so = (size_t)row[k] * SS + c;
          mm[u] = m[so]; vv[u] = v[so]; ww[u] = var[o];
        }
      }
#pragma unroll
      for (int u = 0; u < GK; ++u) {
        const int k = k0 + u, j = k * 32 + lane;
        if (k >= HOLD || row[k] < 0) continue;
        float4 r;
        r.x = dt[u].x + g * (S.x - e[k].x); r.y = dt[u].y + g * (S.y - e[k].y);
        r.z = dt[u].z + g * (S.z - e[k].z); r.w = dt[u].w + g * (S.w - e[k].w);
        const int entry = b * F + j / LPR;
        if (!(s[k] & DUP_FLAG)) {
          const size_t o = (size_t)row[k] * LPR + c, so = (size_t)row[k] * SS + c;
          adam_apply(ww[u], mm[u], vv[u], r, lr_t, b1, b2, eps);
          m[so] = mm[u]; v[so] = vv[u]; var[o] = ww[u];
          if (c == 0) {
            slot[row[k]] = -1;
            if (touched != nullptr) atomicOr(touched + (row[k] >> 5), 1u << (row[k] & 31));
            ++mine;
          }
        } else {
          dup_grads[(size_t)entry * LPR + c] = r;
          if (c == 0) dup_list[atomicAdd(n_dup, 1)] = entry;
        }
      }
    }
  }
  if (n_unique != nullptr) {
    mine = __reduce_add_sync(full, mine);
    if (lane == 0 && mine) atomicAdd(reinterpret_cast<unsigned long long*>(n_unique), (unsigned long long)mine);
  }
}

// list-driven finish of the duplicated rows: MERGE (every non-claiming entry adds its parked values into the claiming entry's)
template <int LPR>
__global__ void __launch_bounds__(256)
adam_dup_merge_kernel(const EntrySrc src, const int* __restrict__ slot, float4* __restrict__ dup_grads,
                      const int* __restrict__ dup_list, const int* __restrict__ n_dup) {
  const size_t total = (size_t)(*n_dup) * LPR;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int e = __ldg(dup_list + t / LPR);
    const long long row = entry_row(src, e);
    const int w = __ldg(slot + row) & ~DUP_FLAG;
    if (w != e) atomicAdd(dup_grads + (size_t)w * LPR + t % LPR, dup_grads[(size_t)e * LPR + t % LPR]);
  }
}
// ... then UPDATE by the claiming entries
template <int LPR>
__global__ void __launch_bounds__(256)
adam_dup_update_kernel(float4* __restrict__ var, float4* __restrict__ m, float4* __restrict__ v, int SS, const EntrySrc src,
                       int* __restrict__ slot, const float4* __restrict__ dup_grads, const int* __restrict__ dup_list,
                       const int* __restrict__ n_dup, float lr_t, float b1, float b2, float eps, unsigned int* __restrict__ touched,
                       long long* __restrict__ n_unique) {
  const size_t total = (size_t)(*n_dup) * LPR;
  int mine = 0;
  for (size_t base = ((size_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31)); base < total; base += (size_t)gridDim.x * blockDim.x) {
    const size_t t = base + (threadIdx.x & 31);
    long long row = -1;
    int e = -1;
    bool win = false;
    if (t < total) {
      e = __ldg(dup_list + t / LPR);
      row = entry_row(src, e);
      win = (slot[row] & ~DUP_FLAG) == e;
    }
    __syncwarp();                      // every lane of an entry has read the slot before its lane 0 clears it
    if (!win) continue;
    const size_t o = (size_t)row * LPR + t % LPR, so = (size_t)row * SS + t % LPR;
    const float4 g = dup_grads[(size_t)e * LPR + t % LPR];
    float4 mm = m[so], vv = v[so], w = var[o];
    adam_apply(w, mm, vv, g, lr_t, b1, b2, eps);
    m[so] = mm; v[so] = vv; var[o] = w;
    if (t % LPR == 0) {
      slot[row] = -1;
      if (touched != nullptr) atomicOr(touched + (row >> 5), 1u << (row & 31));
      ++mine;
    }
  }
  if (n_unique != nullptr) {
    mine = __reduce_add_sync(0xffffffffu, mine);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(reinterpret_cast<unsigned long long*>(n_unique), (unsigned long long)mine);
  }
}

// state_stride: floats between consecutive rows of m (and of v).  D = two separate (V, D) tables; 2*D = ONE interleaved
// (V, 2, D) buffer with v = m + D: a row's two moments then share a DRAM page, which is what the random row updates are
// bound by (measured access-rate limit ~30 G rows/s, DESIGN 4.1) -- 4 instead of 6 row activations per updated row.
static int check_stride(const char* fn, int64_t D, int64_t state_stride) {
  CTR_REQUIRE(state_stride >= D && state_stride % 4 == 0 && state_stride <= (1LL << 20), "%s: state_stride=%lld must be a multiple of 4 and >= D",
              fn, (long long)state_stride);
  return CTR_OK;
}

static int check_adam(const char* fn, int64_t V, int64_t D) {
  CTR_REQUIRE(V >= 0, "%s: bad V", fn);
  CTR_UNSUPPORTED(D % 4 != 0 || D > 128 || (D & (D - 1)) != 0, "%s: D=%lld unsupported (power of two in 4..128)", fn, (long long)D);
  return CTR_OK;
}

}  // namespace ctr

using namespace ctr;

extern "C" int ctr_adam_rows(float* var, float* m, float* v, int64_t state_stride, int64_t V, int64_t D, const int64_t* rows, const float* grads,
                             const int64_t* count, int64_t max_n, float lr_t, float beta1, float beta2, float eps,
                             uint32_t* touched_bitmap, void* stream) {
  int rc = check_adam("ctr_adam_rows", V, D);
  if (rc) return rc;
  if ((rc = check_stride("ctr_adam_rows", D, state_stride))) return rc;
  CTR_REQUIRE(var && m && v && rows && grads && max_n >= 0, "ctr_adam_rows: null argument / bad size");
  CTR_REQUIRE(aligned16(var) && aligned16(m) && aligned16(v) && aligned16(grads), "ctr_adam_rows: buffers must be 16-byte aligned");
  if (max_n == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  const long long total = (long long)max_n * (D / 4);
  const int grid = (int)((total + 255) / 256 < (long long)sm_count() * 16 ? (total + 255) / 256 : (long long)sm_count() * 16);
#define GO(L) adam_rows_kernel<L><<<grid, 256, 0, st>>>(reinterpret_cast<float4*>(var), reinterpret_cast<float4*>(m), reinterpret_cast<float4*>(v), (int)(state_stride / 4), V, reinterpret_cast<const long long*>(rows), reinterpret_cast<const float4*>(grads), reinterpret_cast<const long long*>(count), max_n, lr_t, beta1, beta2, eps, touched_bitmap)
  switch (D / 4) { case 1: GO(1); break; case 2: GO(2); break; case 4: GO(4); break; case 8: GO(8); break; case 16: GO(16); break; default: GO(32); break; }
#undef GO
  CTR_CHECK_LAUNCH("ctr_adam_rows");
  return CTR_OK;
}

extern "C" int ctr_adam_dense_rest(float* var, float* m, float* v, int64_t state_stride, int64_t V, int64_t D, float lr_t, float beta1, float beta2,
                                   float eps, const uint32_t* touched_bitmap, void* stream) {
  int rc = check_adam("ctr_adam_dense_rest", V, D);
  if (rc) return rc;
  if ((rc = check_stride("ctr_adam_dense_rest", D, state_stride))) return rc;
  CTR_REQUIRE(var && m && v, "ctr_adam_dense_rest: null argument");
  CTR_REQUIRE(aligned16(var) && aligned16(m) && aligned16(v), "ctr_adam_dense_rest: buffers must be 16-byte aligned");
  if (V == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  const long long total = (long long)V * (D / 4);
  const int grid = (int)((total + 255) / 256 < (long long)sm_count() * 32 ? (total + 255) / 256 : (long long)sm_count() * 32);
#define GO(L) adam_dense_rest_kernel<L><<<grid, 256, 0, st>>>(reinterpret_cast<float4*>(var), reinterpret_cast<float4*>(m), reinterpret_cast<float4*>(v), (int)(state_stride / 4), V, lr_t, beta1, beta2, eps, touched_bitmap)
  switch (D / 4) { case 1: GO(1); break; case 2: GO(2); break; case 4: GO(4); break; case 8: GO(8); break; case 16: GO(16); break; default: GO(32); break; }
#undef GO
  CTR_CHECK_LAUNCH("ctr_adam_dense_rest");
  return CTR_OK;
}

static int adam_dedup_launch(const char* fn, float* var, float* m, float* v, int64_t state_stride, int64_t D, const EntrySrc& src, long long n,
                             float* vals, int32_t* slot_of_row, int32_t* dup_list, float lr_t, float beta1, float beta2, float eps,
                             uint32_t* touched_bitmap, int64_t* n_unique, cudaStream_t st) {
  const long long total = n * (D / 4);
  auto cap = [](long long want, long long lim) { return (int)(want < lim ? want : lim); };
  const int grid_e = cap((n + 255) / 256, (long long)sm_count() * 16), grid_t = cap((total + 255) / 256, (long long)sm_count() * 16);
  auto* g4 = reinterpret_cast<float4*>(vals);
  if (dup_list != nullptr) {
    CTR_CUDA(cudaMemsetAsync(dup_list + n, 0, sizeof(int32_t), st));
    adam_claim_list_kernel<<<grid_e, 256, 0, st>>>(src, n, slot_of_row, dup_list, dup_list + n);
  } else {
    adam_claim_kernel<<<grid_e, 256, 0, st>>>(src, n, slot_of_row);
  }
#define GO(L)                                                                                                               \
  if (dup_list != nullptr) adam_merge_list_kernel<L><<<sm_count() * 2, 256, 0, st>>>(src, slot_of_row, g4, dup_list, dup_list + n); \
  else adam_merge_kernel<L><<<grid_t, 256, 0, st>>>(src, n, slot_of_row, g4);                                               \
  adam_update_kernel<L><<<grid_t, 256, 0, st>>>(reinterpret_cast<float4*>(var), reinterpret_cast<float4*>(m),               \
                                                reinterpret_cast<float4*>(v), (int)(state_stride / 4), src, n, slot_of_row, g4, lr_t, beta1, beta2,  \
                                                eps, touched_bitmap, reinterpret_cast<long long*>(n_unique))
  switch (D / 4) { case 1: GO(1); break; case 2: GO(2); break; case 4: GO(4); break; case 8: GO(8); break; case 16: GO(16); break; default: GO(32); break; }
#undef GO
  CTR_CHECK_LAUNCH(fn);
  count_launch(2);
  return CTR_OK;
}

extern "C" int ctr_adam_indexed_slices(float* var, float* m, float* v, int64_t state_stride, const int64_t* field_row_offset, int64_t F, int64_t D,
                                       const int64_t* ids, float* row_grads, int64_t B, int32_t* slot_of_row, int32_t* dup_list,
                                       float lr_t, float beta1, float beta2, float eps, uint32_t* touched_bitmap,
                                       int64_t* n_unique, void* stream) {
  int rc = check_adam("ctr_adam_indexed_slices", 0, D);
  if (rc) return rc;
  if ((rc = check_stride("ctr_adam_indexed_slices", D, state_stride))) return rc;
  CTR_REQUIRE(var && m && v && field_row_offset && ids && row_grads && slot_of_row, "ctr_adam_indexed_slices: null argument");
  CTR_REQUIRE(B >= 0 && F >= 1 && F <= (1 << 20) && B * F < (1LL << 30), "ctr_adam_indexed_slices: bad B/F (B*F must be < 2^30)");
  CTR_REQUIRE(aligned16(var) && aligned16(m) && aligned16(v) && aligned16(row_grads),
              "ctr_adam_indexed_slices: buffers must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  EntrySrc src = {reinterpret_cast<const long long*>(ids), reinterpret_cast<const long long*>(field_row_offset), nullptr, 0, 0, (int)F};
  return adam_dedup_launch("ctr_adam_indexed_slices", var, m, v, state_stride, D, src, B * F, row_grads, slot_of_row, dup_list, lr_t, beta1, beta2, eps,
                           touched_bitmap, n_unique, as_stream(stream));
}

extern "C" int ctr_adam_rows_dedup(float* var, float* m, float* v, int64_t state_stride, int64_t V, int64_t D, const int64_t* rows, float* vals,
                                   const int64_t* counts, int64_t nseg, int64_t cap, int32_t* slot_of_row, int32_t* dup_list,
                                   float lr_t, float beta1, float beta2, float eps, uint32_t* touched_bitmap, int64_t* n_unique,
                                   void* stream) {
  int rc = check_adam("ctr_adam_rows_dedup", V, D);
  if (rc) return rc;
  if ((rc = check_stride("ctr_adam_rows_dedup", D, state_stride))) return rc;
  CTR_REQUIRE(var && m && v && rows && vals && counts && slot_of_row, "ctr_adam_rows_dedup: null argument");
  CTR_REQUIRE(nseg >= 1 && cap >= 0 && nseg * cap < (1LL << 30), "ctr_adam_rows_dedup: bad nseg/cap (nseg*cap must be < 2^30)");
  CTR_REQUIRE(aligned16(var) && aligned16(m) && aligned16(v) && aligned16(vals), "ctr_adam_rows_dedup: buffers must be 16-byte aligned");
  if (cap == 0 || V == 0) return CTR_OK;
  EntrySrc src = {reinterpret_cast<const long long*>(rows), nullptr, reinterpret_cast<const long long*>(counts), cap, V, 0};
  return adam_dedup_launch("ctr_adam_rows_dedup", var, m, v, state_stride, D, src, nseg * cap, vals, slot_of_row, dup_list, lr_t, beta1, beta2, eps,
                           touched_bitmap, n_unique, as_stream(stream));
}

template <int LPR, int HOLD>
static int launch_bwd_adam(const float* tile, const float* d_tile, const float* d_fm2, const EntrySrc& src, int64_t B, int64_t F,
                           float* var, float* m, float* v, int SS, int32_t* slot, float* dup_grads, int32_t* dup_list, float lr_t, float b1,
                           float b2, float eps, uint32_t* touched, int64_t* n_unique, cudaStream_t st) {
  auto k = embed_fm2_bwd_adam_kernel<LPR, HOLD>;
  int per_sm = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, 256, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  long long grid = (long long)per_sm * sm_count();
  if (grid > (B + 7) / 8) grid = (B + 7) / 8;
  int* n_dup = dup_list + B * F;
  k<<<(int)grid, 256, 0, st>>>(reinterpret_cast<const float4*>(tile), reinterpret_cast<const float4*>(d_tile), d_fm2, src.off, src.ids,
                               (int)B, (int)F, reinterpret_cast<float4*>(var), reinterpret_cast<float4*>(m),
                               reinterpret_cast<float4*>(v), SS, slot, reinterpret_cast<float4*>(dup_grads), dup_list, n_dup, lr_t, b1, b2,
                               eps, touched, reinterpret_cast<long long*>(n_unique));
  const int g2 = sm_count() * 2;
  adam_dup_merge_kernel<LPR><<<g2, 256, 0, st>>>(src, slot, reinterpret_cast<float4*>(dup_grads), dup_list, n_dup);
  adam_dup_update_kernel<LPR><<<g2, 256, 0, st>>>(reinterpret_cast<float4*>(var), reinterpret_cast<float4*>(m),
                                                  reinterpret_cast<float4*>(v), SS, src, slot, reinterpret_cast<const float4*>(dup_grads),
                                                  dup_list, n_dup, lr_t, b1, b2, eps, touched, reinterpret_cast<long long*>(n_unique));
  CTR_CHECK_LAUNCH("ctr_embed_fm2_bwd_adam");
  count_launch(2);
  return CTR_OK;
}

template <int LPR>
static int dispatch_bwd_adam(const float* tile, const float* d_tile, const float* d_fm2, const EntrySrc& src, int64_t B, int64_t F,
                             float* var, float* m, float* v, int SS, int32_t* slot, float* dup_grads, int32_t* dup_list, float lr_t, float b1,
                             float b2, float eps, uint32_t* touched, int64_t* n_unique, cudaStream_t st) {
  const int64_t per_lane = (F * LPR + 31) / 32;
#define GO(H) return launch_bwd_adam<LPR, H>(tile, d_tile, d_fm2, src, B, F, var, m, v, SS, slot, dup_grads, dup_list, lr_t, b1, b2, eps, touched, n_unique, st)
  if (per_lane <= 4) GO(4);
  if (per_lane <= 8) GO(8);
  if (per_lane <= 12) GO(12);
#undef GO
  set_error("ctr_embed_fm2_bwd_adam: F*D = %lld exceeds the register-resident limit of 1536 (use ctr_embed_fm2_bwd + ctr_adam_indexed_slices)",
            (long long)(F * LPR * 4));
  return CTR_ERR_UNSUPPORTED;
}

extern "C" int ctr_embed_fm2_bwd_adam(const float* tile, const float* d_tile, const float* d_fm2, const int64_t* field_row_offset,
                                      const int64_t* ids, int64_t B, int64_t F, int64_t D, float* var, float* m, float* v,
                                      int64_t state_stride, int32_t* slot_of_row, float* dup_grads, int32_t* dup_list, float lr_t, float beta1, float beta2,
                                      float eps, uint32_t* touched_bitmap, int64_t* n_unique, void* stream) {
  int rc = check_adam("ctr_embed_fm2_bwd_adam", 0, D);
  if (rc) return rc;
  if ((rc = check_stride("ctr_embed_fm2_bwd_adam", D, state_stride))) return rc;
  CTR_REQUIRE(tile && field_row_offset && ids && var && m && v && slot_of_row && dup_grads && dup_list,
              "ctr_embed_fm2_bwd_adam: null argument");
  CTR_REQUIRE(B >= 0 && F >= 1 && F <= 65536 && B * F < (1LL << 30), "ctr_embed_fm2_bwd_adam: bad B/F (B*F must be < 2^30)");
  CTR_REQUIRE(aligned16(tile) && aligned16(d_tile) && aligned16(var) && aligned16(m) && aligned16(v) && aligned16(dup_grads),
              "ctr_embed_fm2_bwd_adam: buffers must be 16-byte aligned");
  if (B == 0) return CTR_OK;
  cudaStream_t st = as_stream(stream);
  EntrySrc src = {reinterpret_cast<const long long*>(ids), reinterpret_cast<const long long*>(field_row_offset), nullptr, 0, 0, (int)F};
  const long long n = (long long)B * F;
  CTR_CUDA(cudaMemsetAsync(dup_list + n, 0, sizeof(int32_t), st));
  const int grid_e = (int)((n + 255) / 256 < (long long)sm_count() * 16 ? (n + 255) / 256 : (long long)sm_count() * 16);
  adam_claim_dup_kernel<<<grid_e, 256, 0, st>>>(src, n, slot_of_row);
  count_launch(1);
  switch (D / 4) {
#define GO(L) case L: return dispatch_bwd_adam<L>(tile, d_tile, d_fm2, src, B, F, var, m, v, (int)(state_stride / 4), slot_of_row, dup_grads, dup_list, lr_t, beta1, beta2, eps, touched_bitmap, n_unique, st)
    GO(1); GO(2); GO(4); GO(8); GO(16);
    default: return dispatch_bwd_adam<32>(tile, d_tile, d_fm2, src, B, F, var, m, v, (int)(state_stride / 4), slot_of_row, dup_grads, dup_list, lr_t, beta1, beta2, eps, touched_bitmap, n_unique, st);
#undef GO
  }
}

/* ctr_b200.h -- C ABI of the Hopper-native (sm_90a) CTR feature-interaction engine (libctr_b200.so).
 *
 * Drop-in boundary for the hot path of tangxyw/RecAlgorithm (reference paths below are relative to
 * the reference's algorithm/ directory).  The reference has no FFI of its own -- its boundary is Python
 * callables invoked while a TF1 graph is built (SURVEY.md section 8b) -- so each entry point here
 * names the reference callable whose forward / autodiff-backward it replaces.  The Python side
 * (recalgorithm_b200/layers.py) re-exposes them under the reference's own signatures.
 *
 * Conventions
 *   - plain C: raw DEVICE pointers, int64_t sizes, `void* stream` is a cudaStream_t (NULL = default stream);
 *   - every function returns 0 on success or a negative CTR_ERR_* code; ctr_last_error() gives the text
 *     (thread-local).  Argument errors are detected before any launch;
 *   - the CALLER owns every buffer; kernels never allocate, never synchronise, and are re-entrant
 *     across streams.  Where a workspace is needed there is a *_workspace_bytes() query;
 *   - all tensors are dense row-major fp32 unless stated; ids / offsets / lengths are int64;
 *   - there is no CPU fallback: on a machine without an sm_90 GPU every compute entry point fails
 *     with CTR_ERR_CUDA.
 */
#ifndef CTR_B200_H_
#define CTR_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTR_OK 0
#define CTR_ERR_INVALID_ARG (-1)
#define CTR_ERR_UNSUPPORTED (-2)
#define CTR_ERR_CUDA (-3)

/* ---- library ---------------------------------------------------------------------------------- */
const char* ctr_last_error(void);
int ctr_version(void);                          /* ABI version, currently 1 */
int ctr_device_info(int* sm_count, int* cc_major, int* cc_minor);   /* current device */
int ctr_enable_peer_access(int peer_device);     /* map `peer_device`'s memory into the current device (NVLink P2P); idempotent */
/* Peer-mappable device buffers for the row-sharded path: a plain device allocation, its 64-byte CUDA-IPC handle, and the
 * import of a peer's handle into the current device's address space (peer access over NVLink is enabled on import). */
int ctr_peer_alloc(int64_t bytes, void** ptr);
int ctr_peer_free(void* ptr);
int ctr_ipc_export(void* ptr, unsigned char* handle64);
int ctr_ipc_import(const unsigned char* handle64, void** ptr);
int ctr_ipc_close(void* ptr);
/* The same role from the CUDA virtual-memory-management API (cuMemCreate / cuMemMap), shared as POSIX file descriptors: the
 * mapping the big table shards use -- a legacy-IPC mapping of a 32 GB shard collapses under random 128-byte peer reads, and
 * with VMM the size / address alignment chosen here (align = 0: the driver's recommended granularity) sets the page size the
 * peers' TLBs see.  ctr_vmm_alloc maps `bytes` (rounded up to `align`) on the current device and returns the fd to hand to
 * the peers (e.g. through pidfd_getfd); ctr_vmm_import maps a peer's fd into the current device (read/write over NVLink). */
int ctr_vmm_granularity(int64_t* minimum, int64_t* recommended);
int ctr_vmm_alloc(int64_t bytes, int64_t align, void** ptr, int* fd, int64_t* mapped_bytes);
int ctr_vmm_import(int fd, int64_t mapped_bytes, int64_t align, void** ptr);
int ctr_vmm_free(void* ptr);
int64_t ctr_kernel_launches(void);              /* kernels launched by this library so far (process-wide) */

/* ---- Row L + FM2: fused embedding lookup + DeepFM second-order term ------------------------------
 * Replaces   fc.input_layer(features, [embedding_column])   x F   (DeepFM/deepfm.py:187-190;
 *            xDeepFM/xdeepfm.py:158,167; DCN/dcn.py:153; FiBiNET/fibinet.py:162-163)
 *   and the inline FM second-order block (DeepFM/deepfm.py:192-200).
 *
 * table            (V_total, D): the F per-field tables stored back to back; field f owns rows
 *                  [field_row_offset[f], field_row_offset[f+1]).
 * field_row_offset device int64[F+1].
 * ids              device int64 (B, F), per-field local ids.  id < 0 (the vocabulary's OOV / '' value, -1)
 *                  or id >= the field's row count gives the ZERO vector (TF: pruned id -> empty bag -> zeros).
 * tile             out (B, F, D) contiguous, or NULL (lookup+FM2 only).
 * fm2              out (B), 0.5 * sum_d[(sum_f e)^2 - sum_f e^2], or NULL (lookup only).
 * D must be a multiple of 4 and <= 128 (128-bit row chunks); other widths go through ctr_bag_lookup_*.
 */
int ctr_embed_fm2_fwd(const float* table, const int64_t* field_row_offset, const int64_t* ids,
                      int64_t B, int64_t F, int64_t D, float* tile, float* fm2, void* stream);
/* The same with int32 ids (half the id bytes over PCIe / HBM); ids64_out (may be NULL) receives the widened (B,F) int64 copy
 * for IndexedSlices consumers (optimizers, ctr_embed_scatter_add). */
int ctr_embed_fm2_fwd_ids32(const float* table, const int64_t* field_row_offset, const int32_t* ids, int64_t B, int64_t F,
                            int64_t D, float* tile, float* fm2, int64_t* ids64_out, void* stream);

/* Sequence lookup: ids (B, T) all index ONE table -- rows [row_range[0], row_range[1]) of `table` (device int64[2]) -- e.g.
 * the padded behaviour history of tf.contrib.feature_column.sequence_input_layer over a shared embedding (DIN/din.py:209-214).
 * out (B, T, D); id < 0 or out of range -> zero row (the zero padding).  One warp per sample, like ctr_embed_fm2_fwd.  Its
 * gradient is the IndexedSlices (ids, d_out) as is -- no kernel. */
int ctr_embed_seq_fwd(const float* table, const int64_t* row_range, const int64_t* ids, int64_t B, int64_t T, int64_t D,
                      float* out, void* stream);

/* Backward of the pair above = the `values` of TF's IndexedSlices gradient of the gather
 * (indices are the caller's ids):   row_grads[b,f,:] = d_tile[b,f,:] + d_fm2[b] * (S[b,:] - e[b,f,:]),
 * S = sum_f e[b,f,:].   tile = the forward output; d_tile (B,F,D) and d_fm2 (B) may each be NULL (= 0).
 * Rows whose id was invalid receive a gradient too (it is simply never applied; see ctr_embed_scatter_add). */
int ctr_embed_fm2_bwd(const float* tile, const float* d_tile, const float* d_fm2,
                      int64_t B, int64_t F, int64_t D, float* row_grads, void* stream);

/* Lookup + FM2 with a fused dense(1) consumer of the flattened tile (the first use of the tile by DeepFM's deep part,
 * DeepFM/deepfm.py:203-212, reduced to one unit): lin[b] = sum_{f,d} tile[b,f,d]*wlin[f,d].  ids: int64 (ids_are_int32 = 0)
 * or int32 (= 1; ids64_out, may be NULL, receives the widened copy).  tile may be NULL only if no backward follows. */
int ctr_embed_fm2_lin_fwd(const float* table, const int64_t* field_row_offset, const void* ids, int ids_are_int32, int64_t B,
                          int64_t F, int64_t D, const float* wlin, float* tile, float* fm2, float* lin, int64_t* ids64_out,
                          void* stream);
/* Its backward: the upstream gradient of the tile is the rank-1 product d_lin[b]*wlin[f,d] and is never materialised:
 *   row_grads[b,f,:] = d_lin[b]*wlin[f,:] + d_fm2[b]*(S[b,:] - e[b,f,:]);   d_wlin[f,:] = sum_b d_lin[b]*e[b,f,:]
 * (d_wlin (F*D) is zeroed here; fp32 atomics across CTAs).  F*D <= 1536. */
int ctr_embed_fm2_lin_bwd(const float* tile, const float* wlin, const float* d_fm2, const float* d_lin, int64_t B, int64_t F,
                          int64_t D, float* row_grads, float* d_wlin, void* stream);

/* Mean sigmoid cross-entropy of logits = logit_a (+ logit_b, may be NULL) against labels, (B) each, and its gradient in one
 * launch: *loss = mean_b[max(x,0) - x*z + log1p(exp(-|x|))] (tf.nn.sigmoid_cross_entropy_with_logits + reduce_mean,
 * DeepFM/deepfm.py:214,235), d_logit[b] = (sigmoid(x) - z)/B (may be NULL).  fp32 atomics across CTAs for the mean. */
int ctr_sigmoid_ce(const float* logit_a, const float* logit_b, const float* labels, int64_t B, float* loss, float* d_logit,
                   void* stream);

/* Densify: grad_table[field_row_offset[f] + ids[b,f], :] += row_grads[b,f,:] for valid ids (duplicates
 * summed, like the optimizer's IndexedSlices de-duplication; TF-internal, SURVEY A.8).  grad_table is
 * NOT zeroed here.  fp32 red.global.add -> summation order is not deterministic. */
int ctr_embed_scatter_add(float* grad_table, const int64_t* field_row_offset, const int64_t* ids,
                          const float* row_grads, int64_t B, int64_t F, int64_t D, void* stream);

/* ---- Row (e): row-sharded tables across the GPUs of one NVSwitch box -----------------------------------------
 * Global row gr = field_row_offset[f] + id is owned by rank gr % G and stored at local row gr / G (G a power of two <= 8).
 * The reference has no multi-device path; the semantics kept are the lookup's and the IndexedSlices gradient's.
 *
 * Forward: same contract as ctr_embed_fm2_fwd, but rows are PULLED from the owners' shards inside the gather kernel.
 * shard_ptrs: HOST array of G device pointers, entry r = rank r's shard (ceil(V_total/G), D) as mapped into THIS process
 * (CUDA IPC / peer mapping for r != own rank).  No collective is involved. */
int ctr_embed_fm2_fwd_sharded(const float* const* shard_ptrs, int64_t G, const int64_t* field_row_offset,
                              const int64_t* ids, int64_t B, int64_t F, int64_t D, float* tile, float* fm2, void* stream);
/* The same with int32 ids (half the id bytes over PCIe / HBM); ids64_out (may be NULL) receives the widened (B,F) int64 copy
 * that IndexedSlices consumers downstream expect. */
int ctr_embed_fm2_fwd_sharded_ids32(const float* const* shard_ptrs, int64_t G, const int64_t* field_row_offset,
                                    const int32_t* ids, int64_t B, int64_t F, int64_t D, float* tile, float* fm2,
                                    int64_t* ids64_out, void* stream);
/* Sharded form of ctr_embed_fm2_lin_fwd (fused dense(1) head; rows pulled from the owners' shards). */
int ctr_embed_fm2_lin_fwd_sharded(const float* const* shard_ptrs, int64_t G, const int64_t* field_row_offset, const void* ids,
                                  int ids_are_int32, int64_t B, int64_t F, int64_t D, const float* wlin, float* tile, float* fm2,
                                  float* lin, int64_t* ids64_out, void* stream);
/* Gradient exchange, step 1 (independent of the forward; one pass over the ids): assigns every valid (b,f) a slot in its
 * OWNER's receive queue and writes plan[b,f] = owner << 28 | slot (-1: invalid id, or dropped because the owner's slice is
 * full -> *overflow = 1).  The queue's local-row indices are written here, as contiguous runs per owner:
 * recv_rows / recv_counts: HOST arrays of G device pointers; entry d = owner d's (G_src, capacity) int64 row queue /
 * (G_src,) int64 count vector as mapped into this process; this rank writes slice [my_rank] and, when the kernel ends,
 * recv_counts[d][my_rank] = min(entries queued at d, capacity) (recv_counts or its entries may be NULL).
 * ids: int64 (ids_are_int32 = 0) or int32 (= 1).
 * counters: device int64[9] scratch, zeroed here (ends as entries per owner + a ticket); overflow: device int, zeroed here.
 * B*F < 2^28, capacity < 2^28. */
int ctr_sharded_plan(const int64_t* field_row_offset, const void* ids, int ids_are_int32, int64_t B, int64_t F, int64_t G, int64_t my_rank,
                     int64_t* const* recv_rows, int64_t* const* recv_counts, int64_t capacity, int64_t* counters,
                     int* overflow, int32_t* plan, void* stream);
/* Gradient exchange, step 2, fused into the lookup backward: same arithmetic as ctr_embed_fm2_bwd, but every planned row of
 * d_tile + d_fm2*(S - e) is stored straight into its owner's value queue with 128-bit peer stores (recv_vals: HOST array of
 * G device pointers, entry d = owner d's (G_src, capacity, D) fp32 queue; slice [my_rank] is written).  row_grads may be
 * NULL: the IndexedSlices values then never touch local HBM.  Follow with a stream sync and a cross-rank barrier before
 * any owner reads its queues. */
int ctr_embed_fm2_bwd_push(const float* tile, const float* d_tile, const float* d_fm2, const int32_t* plan, int64_t B,
                           int64_t F, int64_t D, int64_t G, int64_t my_rank, float* const* recv_vals, int64_t capacity,
                           float* row_grads, void* stream);
/* The same for the fused dense(1) head (ctr_embed_fm2_lin_fwd_sharded): d_tile is the rank-1 product d_lin[b]*wlin[f,d] and is
 * never materialised; d_wlin (F*D, zeroed here) = sum_b d_lin[b]*tile[b].  F*D <= 1536. */
int ctr_embed_fm2_lin_bwd_push(const float* tile, const float* wlin, const float* d_fm2, const float* d_lin, const int32_t* plan,
                               int64_t B, int64_t F, int64_t D, int64_t G, int64_t my_rank, float* const* recv_vals,
                               int64_t capacity, float* row_grads, float* d_wlin, void* stream);
/* The exchange alone, for row gradients (B,F,D) produced by any other backward. */
int ctr_sharded_grad_push(const float* row_grads, const int32_t* plan, int64_t B, int64_t F, int64_t D, int64_t G,
                          int64_t my_rank, float* const* recv_vals, int64_t capacity, void* stream);
/* Owner side / generic IndexedSlices consumer: dst[rows[i], :] += vals[i, :] for i < min(*count, max_n) (count may be
 * NULL = max_n); rows outside [0, V) are ignored.  fp32 vector red.global.add. */
int ctr_rows_scatter_add(float* dst, int64_t V, int64_t D, const int64_t* rows, const float* vals, const int64_t* count,
                         int64_t max_n, void* stream);

/* ---- SURVEY 8f.3: Adam on the IndexedSlices gradient of a table (the step right after the hot path) ------------------
 * Reference: tf.train.AdamOptimizer(lr, .9, .999, 1e-8) (DeepFM/deepfm.py:246-250); its sparse apply sums duplicate
 * indices, decays m and v of the WHOLE table and updates every row (SURVEY A.8); DIEN uses LazyAdam (DIEN/dien.py:328).
 * rows (n) must be UNIQUE with grads (n, D) already summed per row (ctr_rows_scatter_add into a compact buffer does that);
 * lr_t = lr*sqrt(1-beta2^t)/(1-beta1^t) is computed by the caller.  count: device int64 (NULL = max_n).
 * state_stride (all ctr_adam_* entry points) = floats between consecutive rows of m (and of v): D for two separate (V, D)
 * tables, 2*D for ONE interleaved (V, 2, D) buffer with v = m + D -- a row's two moments then share a DRAM page, which is
 * what the random row updates are bound by (4 instead of 6 row activations per updated row).
 * ctr_adam_rows updates m, v, var of the listed rows (and sets their bit in touched_bitmap (ceil(V/32) uint32, zeroed by
 * the caller) when given) = LazyAdam; ctr_adam_dense_rest then applies the g = 0 update to every row whose bit is clear
 * = the reference's dense semantics. */
int ctr_adam_rows(float* var, float* m, float* v, int64_t state_stride, int64_t V, int64_t D, const int64_t* rows, const float* grads,
                  const int64_t* count, int64_t max_n, float lr_t, float beta1, float beta2, float eps,
                  uint32_t* touched_bitmap, void* stream);
int ctr_adam_dense_rest(float* var, float* m, float* v, int64_t state_stride, int64_t V, int64_t D, float lr_t, float beta1, float beta2, float eps,
                        const uint32_t* touched_bitmap, void* stream);

/* Fused IndexedSlices step (no sort, no host round trip): ids (B,F) per-field local ids (out-of-range = skipped, like the
 * lookup), row_grads (B,F,D) = the IndexedSlices values of ctr_embed_fm2_bwd -- CONSUMED (duplicates of a row are summed
 * into one of its entries).  slot_of_row: int32 per table row, all -1 on entry and again on exit (persistent scratch of
 * the optimizer).  Applies the LazyAdam update to every referenced row with the SUMMED gradient (TF sums duplicates
 * first); sets the rows' bits in touched_bitmap when given (then ctr_adam_dense_rest completes tf.train.AdamOptimizer's
 * dense semantics); adds the number of distinct rows to *n_unique when given.  dup_list: int32[B*F + 1] scratch or NULL --
 * when given, the claim pass lists the entries that met an already claimed row and the merge walks that list instead of
 * re-scanning every entry.  B*F < 2^30. */
int ctr_adam_indexed_slices(float* var, float* m, float* v, int64_t state_stride, const int64_t* field_row_offset, int64_t F, int64_t D,
                            const int64_t* ids, float* row_grads, int64_t B, int32_t* slot_of_row, int32_t* dup_list,
                            float lr_t, float beta1, float beta2, float eps, uint32_t* touched_bitmap, int64_t* n_unique,
                            void* stream);

/* Lookup backward FUSED with that step (SURVEY 8f.3: the row update without writing row-grads to HBM): computes the
 * IndexedSlices values d_tile + d_fm2*(S - e) of ctr_embed_fm2_bwd in registers and applies the LazyAdam update to every row
 * referenced ONCE in the batch on the spot; rows referenced several times park their values in dup_grads ((B,F,D) scratch,
 * written sparsely) and their entry in dup_list (int32[B*F + 1] scratch, last element = count) and are finished with the
 * SUMMED gradient by two list-driven launches.  slot_of_row / touched_bitmap / n_unique as in ctr_adam_indexed_slices.
 * F*D <= 1536, B*F < 2^30.  Same results as ctr_embed_fm2_bwd followed by ctr_adam_indexed_slices. */
int ctr_embed_fm2_bwd_adam(const float* tile, const float* d_tile, const float* d_fm2, const int64_t* field_row_offset,
                           const int64_t* ids, int64_t B, int64_t F, int64_t D, float* var, float* m, float* v,
                           int64_t state_stride, int32_t* slot_of_row, float* dup_grads, int32_t* dup_list, float lr_t, float beta1, float beta2,
                           float eps, uint32_t* touched_bitmap, int64_t* n_unique, void* stream);

/* The same step for the OWNER side of a row-sharded table: entries are the receive queues filled by ctr_sharded_grad_push --
 * rows (nseg, cap) local row ids, vals (nseg, cap, D) (consumed), counts (nseg,) filled slots per segment; duplicates of a
 * row across and inside segments are summed before the update.  dup_list: int32[nseg*cap + 1] scratch or NULL.
 * nseg*cap < 2^30. */
int ctr_adam_rows_dedup(float* var, float* m, float* v, int64_t state_stride, int64_t V, int64_t D, const int64_t* rows, float* vals,
                        const int64_t* counts, int64_t nseg, int64_t cap, int32_t* slot_of_row, int32_t* dup_list, float lr_t,
                        float beta1, float beta2, float eps, uint32_t* touched_bitmap, int64_t* n_unique, void* stream);

/* DeepFM first-order ("wide") term as a D=1 lookup (SURVEY 8f.1).  Replaces indicator_column multi-hot (B, sum V) @
 * dense(1) (DeepFM/deepfm.py:72-80,180-181): out[b] = bias + sum_f w[field_row_offset[f] + ids[b,f]]; invalid ids add 0.
 * w (V_total) is the dense(1) kernel; its gradient is the IndexedSlices (ids, d_out[b] broadcast over F) -- no kernel
 * needed -- and d_bias = sum_b d_out[b]. */
int ctr_first_order_fwd(const float* w, const int64_t* field_row_offset, const int64_t* ids, int64_t B, int64_t F,
                        float bias, float* out, void* stream);

/* ---- Wide & Deep wide part: hashed crossed column @ dense(1), FTRL-Proximal --------------------------
 * Replaces indicator_column(crossed_column([userid, manual_tag_list], hash_bucket_size=100000)) -> fc.input_layer ->
 * tf.layers.dense(wide_input, 1) (WideAndDeep/wide_and_deep.py:121-122,208-210) without the (B, num_buckets) multi-hot.
 * values (nnz) int64 vocabulary ids of the K keys (OOV -1 is hashed like any id); offsets (K, B+1) int64: key k of sample b is
 * values[offsets[k,b] : offsets[k,b+1]].  The crosses of b are the Cartesian product of its keys' values, last key fastest
 * (none if a key is empty); the bucket of (v_1..v_K) is  h = hash_key; h = FingerprintCat64(h, (uint64) v_k) for each k;
 * h % num_buckets  (SURVEY A.11; TF's default hash_key is 0xDECAFCAFFE).
 * Forward: out[b] = *bias + sum over b's crosses of kernel[bucket] (duplicates count); bias is read on the device.
 * Backward: d_kernel (num_buckets) is OVERWRITTEN with the dense gradient multi_hot^T d_logit; d_bias (1), optional, with
 * sum_b d_logit[b].  2 <= K <= 4 and 2 <= num_buckets < 2^31, else CTR_ERR_UNSUPPORTED.  B = 0 launches no kernel (the
 * backward still zeroes d_kernel and d_bias). */
int ctr_crossed_indicator_fwd(const int64_t* values, const int64_t* offsets, int64_t K, int64_t B, int64_t num_buckets,
                              uint64_t hash_key, const float* kernel, const float* bias, float* out, void* stream);
int ctr_crossed_indicator_bwd(const int64_t* values, const int64_t* offsets, int64_t K, int64_t B, int64_t num_buckets,
                              uint64_t hash_key, const float* d_logit, float* d_kernel, float* d_bias, void* stream);
/* TF's dense ApplyFtrl (tf.train.FtrlOptimizer, wide_and_deep.py:254-257; SURVEY A.12) on n elements, in place:
 *   new_accum = accum + g^2;  linear += g - (new_accum^-p - accum^-p) / lr * var;  y = new_accum^-p / lr + 2 l2;
 *   var = |linear| > l1 ? (l1 sign(linear) - linear) / y : 0;  accum = new_accum          (p = lr_power; sqrt at p = -0.5)
 * lr > 0, lr_power <= 0, l1 >= 0 and l2 >= 0 as TF takes them, else CTR_ERR_INVALID_ARG.  Any float-aligned buffers: the pass
 * is 128-bit wide when the four share their offset within 16 bytes, element-wise otherwise. */
int ctr_ftrl_apply(float* var, float* accum, float* linear, const float* grad, int64_t n, float lr, float lr_power, float l1,
                   float l2, void* stream);

/* ---- Row L (general): multi-valued bag lookup, combiner='mean' ----------------------------------
 * Replaces fc.input_layer over embedding_column(col, D, combiner='mean') on a VarLen feature
 * (DCN/dcn.py:98,103; xDeepFM/xdeepfm.py:103,108) and any single-valued column whose D is not a
 * multiple of 4 (DCN/dcn.py:99-102 use D = 2 and 4).
 * ids (nnz) flat values, offsets (B+1) CSR; ids < 0 or >= V are dropped; empty bag -> zeros.
 * out[b*out_stride + 0..D) is written (lets the caller place the field inside a (B, sum_d) row). */
int ctr_bag_lookup_fwd(const float* table, int64_t V, int64_t D, const int64_t* ids, const int64_t* offsets,
                       int64_t B, float* out, int64_t out_stride, void* stream);
/* row_grads (nnz, D): d_out[b]/count_b for valid ids, 0 for dropped ids. */
int ctr_bag_lookup_bwd(const float* d_out, int64_t out_stride, int64_t V, int64_t D, const int64_t* ids,
                       const int64_t* offsets, int64_t B, float* row_grads, void* stream);

/* ---- Row CROSS: DCN cross-layer stack --------------------------------------------------------------
 * Replaces the loop `for i: cross_vec = cross_layer(x0, cross_vec, i)` (DCN/dcn.py:157-160) over
 * cross_layer (DCN/cross_layer.py:21-24):  x_{l+1} = x0 * (x_l . w_l) + b_l + x_l,  x_0 = x0.
 * x0 (B,d); w, b (L,d) = the L (d,1) variables wl_i / bl_i stacked; out (B,d) = x_L.
 * xl_in: optional (B,d) start vector (NULL = x0); lets a single layer be called as cross_layer(x0, xl, i). */
int ctr_cross_fwd(const float* x0, const float* xl_in, const float* w, const float* b,
                  int64_t B, int64_t d, int64_t L, float* out, void* stream);
/* Gradients given g_out = dL/dx_L.  dx0 (B,d) receives the gradient through every use of x0
 * (and through x_0 when xl_in == NULL); dxl_in (B,d) is written only when xl_in != NULL.
 * dw, db (L,d) are overwritten (batch-reduced with fp32 atomics across CTAs). */
int ctr_cross_bwd(const float* x0, const float* xl_in, const float* w, const float* b, const float* g_out,
                  int64_t B, int64_t d, int64_t L, float* dx0, float* dxl_in, float* dw, float* db, void* stream);
/* Lookup FUSED with the cross stack: `net = fc.input_layer(features, cols)` (DCN/dcn.py:153) followed by the loop over
 * cross_layer (DCN/dcn.py:157-160) for uniform-width embedding columns.  table / field_row_offset / ids as in
 * ctr_embed_fm2_fwd (ids int64, or int32 when ids_are_int32 != 0; invalid ids give the zero vector); d = F*D.
 * x0 (B, F*D) receives the gathered input (the backward needs it; the lookup backward of a plain gather is the view
 * dx0 -> (B,F,D), no kernel), out (B, F*D) = x_L.  Needs D % 4 == 0, F*D <= 512, L <= 4 (CTR_ERR_UNSUPPORTED otherwise: call
 * ctr_embed_fm2_fwd + ctr_cross_fwd). */
int ctr_embed_cross_fwd(const float* table, const int64_t* field_row_offset, const void* ids, int ids_are_int32,
                        int64_t B, int64_t F, int64_t D, const float* w, const float* b, int64_t L, float* x0, float* out,
                        void* stream);

/* ---- Row CROSS-V2: DCN-V2 cross network ----------------------------------------------------------------
 * The cross network of DCN-V2 (Wang et al., WWW 2021, arXiv:2008.13535, eq. 1-2).  The reference tree has no DCN-V2 code,
 * so this row follows the paper and is checked against a float64 restatement of it.  Row-vector form, l = 0 .. L-1:
 *   x_{l+1} = x0 * z_l + x_l,  z_l = x_l . W_l + b_l    x0 (B,d); x_0 = xl_in (B,d), or x0 when xl_in == NULL;
 *   full rank (rank == 0):  W_l = w[l]          w (L,d,d); u is not read and may be NULL;
 *   low rank (rank >= 1):   W_l = w[l] . u[l]   w (L,d,rank), u (L,rank,d) (the paper's V_l and U_l^T);
 *   b (L,d); out (B,d) = x_L.
 * fp32-class accuracy (3xTF32 on the tensor cores).  1 <= d <= 512, 1 <= L <= 8, 0 <= rank <= 128 (CTR_ERR_UNSUPPORTED
 * otherwise); rows need no alignment; B = 0 launches nothing.  The entries never allocate or synchronise.
 * saved: caller-owned, ctr_cross_v2_workspace_bytes' saved_bytes = B * ((2L - 1) d + L rank) * 4 bytes: the layer inputs
 *   x_1 .. x_{L-1} (L-1, B, d), then z_0 .. z_{L-1} (L, B, d), then at low rank t_l = x_l . w[l] (L, B, rank).  The forward
 *   writes it and the backward reads it.  A forward-only caller may pass saved = NULL (the layers then run in place in out).
 * workspace: 128-byte aligned, at least the workspace_bytes of ctr_cross_v2_workspace_bytes(0, ..) for the forward (the
 *   prepped tf32 weight copies) and of ctr_cross_v2_workspace_bytes(B, ..) for the backward (also dz, dt at low rank and
 *   up to two dx_l, (B, d rounded up to 32), (B, rank rounded up to 32) and (B, d) each).
 * The backward takes g_out = dL/dout (B,d).  dx0 (B,d) receives every use of x0 (and x_0 itself when xl_in == NULL);
 * dxl_in (B,d) is written when xl_in != NULL.  dw, du (not touched at rank 0, may be NULL) and db are overwritten (zeros
 * at B = 0; batch-reduced with fp32 atomics). */
int ctr_cross_v2_workspace_bytes(int64_t B, int64_t d, int64_t L, int64_t rank, int64_t* workspace_bytes,
                                 int64_t* saved_bytes);
int ctr_cross_v2_fwd(const float* x0, const float* xl_in, const float* w, const float* u, const float* b, int64_t B,
                     int64_t d, int64_t L, int64_t rank, float* out, void* saved, void* workspace, int64_t workspace_bytes,
                     void* stream);
int ctr_cross_v2_bwd(const float* x0, const float* xl_in, const float* w, const float* u, const float* b, const void* saved,
                     const float* g_out, int64_t B, int64_t d, int64_t L, int64_t rank, float* dx0, float* dxl_in,
                     float* dw, float* du, float* db, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- Row CROSS-MIX: DCN-Mix cross network (mixture of low-rank cross experts) ---------------------------------
 * DCN-Mix (Wang et al., WWW 2021, arXiv:2008.13535, eq. 3-4), the paper's mixture of K low-rank experts per cross layer.
 * The reference tree has no DCN-Mix code, so this row follows the paper and is checked against a float64 restatement of
 * it.  Row-vector form, l = 0 .. L-1, experts i = 1 .. K, x_0 = x0, g = tanh (activation 1) or the identity (0):
 *   q_i = x_l . v[l,i],  t_i = g(q_i),  m_i = t_i . c[l,i],  c~_i = g(m_i)     v (L,K,d,r) (the paper's V_i^l),
 *                                                                             c (L,K,r,r) (the paper's (C_i^l)^T);
 *   p = softmax_i(x_l . gate) (max subtracted)                                gate (d,K), no bias, shared by all layers;
 *   z_l = sum_i p_i c~_i . u[l,i] + b[l],  x_{l+1} = x0 * z_l + x_l           u (L,K,r,d) (the paper's (U_i^l)^T), b (L,d);
 *   out (B,d) = x_L.  The paper's sum_i p_i (x0 * (c~_i u_i + b)) is this, since sum_i p_i = 1.
 * With K = 1, the identity and c = I, the layer is row CROSS-V2's low-rank layer (w = v[:,0], u = u[:,0]).
 * fp32-class accuracy (3xTF32 on the tensor cores).  1 <= d <= 512, 1 <= L <= 8, 1 <= K <= 16, r >= 1, K*r <= 128
 * (CTR_ERR_UNSUPPORTED otherwise); rows need no alignment; B = 0 launches nothing.  The entries never allocate or
 * synchronise.
 * saved: caller-owned, ctr_cross_mix_workspace_bytes' saved_bytes = B * ((2L - 1) d + L (2 K r + K)) * 4 bytes: the layer
 *   inputs x_1 .. x_{L-1} (L-1, B, d), then z_0 .. z_{L-1} (L, B, d), then t (L, B, K r), c~ (L, B, K r) and p (L, B, K),
 *   experts side by side.  The forward writes it and the backward reads it.  A forward-only caller may pass saved = NULL
 *   (the layers then run in place in out).
 * workspace: 128-byte aligned, at least the workspace_bytes of ctr_cross_mix_workspace_bytes(0, ..) for the forward (the
 *   prepped tf32 weight copies) and of ctr_cross_mix_workspace_bytes(B, ..) for the backward (also its per-sample rows).
 * The backward takes g_out = dL/dout (B,d).  dx0 (B,d) receives every use of x0.  dv, dc, du, db and dgate are
 *   overwritten (zeros at B = 0; batch-reduced with fp32 atomics); dgate sums over the layers. */
int ctr_cross_mix_workspace_bytes(int64_t B, int64_t d, int64_t L, int64_t K, int64_t r, int64_t* workspace_bytes,
                                  int64_t* saved_bytes);
int ctr_cross_mix_fwd(const float* x0, const float* v, const float* c, const float* u, const float* b, const float* gate,
                      int64_t B, int64_t d, int64_t L, int64_t K, int64_t r, int activation, float* out, void* saved,
                      void* workspace, int64_t workspace_bytes, void* stream);
int ctr_cross_mix_bwd(const float* x0, const float* v, const float* c, const float* u, const float* b, const float* gate,
                      const void* saved, const float* g_out, int64_t B, int64_t d, int64_t L, int64_t K, int64_t r,
                      int activation, float* dx0, float* dv, float* dc, float* du, float* db, float* dgate, void* workspace,
                      int64_t workspace_bytes, void* stream);

/* ---- Row CIN: xDeepFM compressed-interaction layer -------------------------------------------------
 * Replaces cin_layer(x0, xk, hk_1, index) (xDeepFM/cin_layer.py:17-30):
 *   out[b,n,d] = sum_{i,j} xk[b,i,d] * x0[b,j,d] * filter[i*m + j, n]
 * x0 (B,m,D); xk (B,hk,D); filter (hk*m, H) = the conv1d filter (1, hk*m, hk_1)[0]; out (B,H,D);
 * pooled (B,H) = sum_d out (the reduce_sum of xDeepFM/xdeepfm.py:173) or NULL.
 * precision: 0 = fp32-class (3xTF32 split on the tensor cores; default, meets 1e-5),
 *            1 = single-pass TF32 (about 1e-3; for speed comparisons only).
 * workspace: ctr_cin_fwd_workspace_bytes() bytes, 128-byte aligned (holds the filter re-ordered / tf32-split for
 *            TMA); may be NULL when that query returns 0 (shapes served by the CUDA-core path). */
int64_t ctr_cin_fwd_workspace_bytes(int64_t B, int64_t m, int64_t hk, int64_t D, int64_t H);
int ctr_cin_fwd(const float* x0, const float* xk, const float* filter, int64_t B, int64_t m, int64_t hk,
                int64_t D, int64_t H, float* out, float* pooled, int precision,
                void* workspace, int64_t workspace_bytes, void* stream);
/* Gradients of ctr_cin_fwd given g_out (B,H,D); dx0 (B,m,D), dxk (B,hk,D), dfilter (hk*m,H) are overwritten. */
int ctr_cin_bwd(const float* x0, const float* xk, const float* filter, const float* g_out,
                int64_t B, int64_t m, int64_t hk, int64_t D, int64_t H,
                float* dx0, float* dxk, float* dfilter,
                void* workspace, int64_t workspace_bytes, void* stream);
int64_t ctr_cin_bwd_workspace_bytes(int64_t B, int64_t m, int64_t hk, int64_t D, int64_t H);

/* ---- PNN product layer (IPNN / OPNN) ---------------------------------------------------------------
 * Replaces the product layer of pnn_model_fn (PNN/pnn.py:125-181):
 *   out = relu(e_flat . wlin + lp + bias)  (B,N),  e (B, F*K) = the fields' embeddings concatenated (field f = columns
 *   f*K .. f*K+K-1), wlin (F*K, N) = linear_part/linear_w, bias (N,);
 *   method 0 = IPNN: wprod = product_part/inner_product_w theta (N,F),  lp[b,n] = sum_k (sum_f theta[n,f] e[b,f,k])^2;
 *   method 1 = OPNN: wprod = product_part/outer_product_w W (N,K,K), s = sum_f e_f,
 *                    lp[b,n] = sum_kl s_k s_l W[n, min(k,l), max(k,l)]   (only the upper triangle of each W_n is read).
 * fp32-class accuracy (3xTF32 on the tensor cores where F*K + Q + 1 <= 128, Q = F(F+1)/2 (IPNN) or K(K+1)/2 (OPNN), and
 * N % 4 == 0; CUDA-core kernels otherwise).  workspace: ctr_pnn_workspace_bytes() bytes, 128-byte aligned; it holds the
 * derived weights and the weight-gradient accumulator.  The backward takes the forward's out (its relu mask) and g_out
 * (B,N) -- 16-byte aligned on the tensor path -- and overwrites d_e (B, F*K), d_wlin (F*K, N), d_wprod (the shape of
 * wprod; the strictly lower triangle of each OPNN W_n gets exactly 0) and d_bias (N,). */
int ctr_pnn_workspace_bytes(int64_t F, int64_t K, int64_t N, int method, int64_t* bytes);
int ctr_pnn_fwd(const float* e, const float* wlin, const float* wprod, const float* bias, int64_t B, int64_t F, int64_t K,
                int64_t N, int method, float* out, void* workspace, int64_t workspace_bytes, void* stream);
int ctr_pnn_bwd(const float* e, const float* wlin, const float* wprod, const float* out, const float* g_out, int64_t B,
                int64_t F, int64_t K, int64_t N, int method, float* d_e, float* d_wlin, float* d_wprod, float* d_bias,
                void* workspace, int64_t workspace_bytes, void* stream);

/* ---- DeepCrossing residual unit -------------------------------------------------------------------------
 * Replaces residual_unit(input, internal_dim, index) (DeepCrossing/residual_unit.py:4-21, looped at
 * DeepCrossing/deepcrossing.py:149-153):
 *   out = relu(x + relu(x . w0 + b0) . w1 + b1)   x (B,d); w0 = dense_{index}_0/kernel (d,H), b0 (H);
 *                                                  w1 = dense_{index}_1/kernel (H,d), b1 (d); out (B,d).
 * fp32-class accuracy (3xTF32 on the tensor cores); the (B,H) hidden activation of the forward stays on chip.
 * d <= 128 and 1 <= H <= 1024 (CTR_ERR_UNSUPPORTED otherwise); B = 0 launches nothing.
 * workspace: 128-byte aligned, at least ctr_residual_unit_workspace_bytes(0, d, H) bytes for the forward (the prepped
 * weights) and ctr_residual_unit_workspace_bytes(B, d, H) for the backward (also h and its gradient, (B,H) each).
 * The backward takes the forward's out (its relu mask) and g_out (B,d), and overwrites d_x (B,d), d_w0 (d,H), d_b0 (H),
 * d_w1 (H,d) and d_b1 (d) (zeros at B = 0).  b1 is not read by the backward. */
int ctr_residual_unit_workspace_bytes(int64_t B, int64_t d, int64_t H, int64_t* bytes);
int ctr_residual_unit_fwd(const float* x, const float* w0, const float* b0, const float* w1, const float* b1, int64_t B,
                          int64_t d, int64_t H, float* out, void* workspace, int64_t workspace_bytes, void* stream);
int ctr_residual_unit_bwd(const float* x, const float* w0, const float* b0, const float* w1, const float* b1,
                          const float* out, const float* g_out, int64_t B, int64_t d, int64_t H, float* d_x, float* d_w0,
                          float* d_b0, float* d_w1, float* d_b1, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- AutoInt interacting layer ---------------------------------------------------------------------------
 * Multi-head self-attention over fields (Song et al., CIKM 2019, arXiv:1810.11921, eq. 5-8).  The reference tree has no
 * AutoInt code (its README lists AutoInt as a to-do), so this row follows the paper and is checked against a float64
 * restatement of it:
 *   Q = x . w_query, K = x . w_key, V = x . w_value, R = x . w_res   x (B,F,d); each w (d, H*dk), head h = columns
 *                                                                    h*dk .. h*dk+dk-1; no biases;
 *   A_h = softmax_j(Q_h[i] . K_h[j])  (no 1/sqrt(dk) scaling),  out = relu(concat_h A_h V_h + R)   out (B,F,H*dk).
 * fp32-class accuracy (3xTF32 on the tensor cores); Q, K, V, R and the scores of the forward stay on chip.
 * 1 <= F <= 64, 1 <= d <= 128, 1 <= dk <= 64, 1 <= H <= 8, H*dk <= 128 (CTR_ERR_UNSUPPORTED otherwise); B = 0 launches
 * nothing.  workspace: 128-byte aligned, at least ctr_autoint_workspace_bytes(0, F, d, H, dk) bytes for the forward (the
 * prepped weights) and ctr_autoint_workspace_bytes(B, F, d, H, dk) for the backward (also the projection gradients,
 * (B*F, 4*H*dk)).  The backward takes the forward's out (its relu mask) and g_out (B,F,H*dk), and overwrites d_x (B,F,d)
 * and the four weight gradients (zeros at B = 0). */
int ctr_autoint_workspace_bytes(int64_t B, int64_t F, int64_t d, int64_t H, int64_t dk, int64_t* bytes);
int ctr_autoint_fwd(const float* x, const float* w_query, const float* w_key, const float* w_value, const float* w_res,
                    int64_t B, int64_t F, int64_t d, int64_t H, int64_t dk, float* out, void* workspace,
                    int64_t workspace_bytes, void* stream);
int ctr_autoint_bwd(const float* x, const float* w_query, const float* w_key, const float* w_value, const float* w_res,
                    const float* out, const float* g_out, int64_t B, int64_t F, int64_t d, int64_t H, int64_t dk, float* d_x,
                    float* d_w_query, float* d_w_key, float* d_w_value, float* d_w_res, void* workspace,
                    int64_t workspace_bytes, void* stream);

/* ---- MMoE expert-gate layer ------------------------------------------------------------------------------
 * Replaces the experts / gates / tower blocks of mmoe_model_fn (MMOE/mmoe.py:207-236) up to the task towers:
 *   h_e     = relu(x . w_e + b_e)        x (B,d) = concat_all_input; w_experts (E,d,H): w_e = experts/expert_{e}/kernel,
 *                                        b_experts (E,H): b_e = experts/expert_{e}/bias, e < E = num_experts;
 *   p_t     = softmax_e(x . g_t)         w_gates (T,d,E): g_t = gates/gate_{t}/kernel (no bias), t < T = num_tasks;
 *   tower_t = sum_e p_t[e] h_e           towers (T,B,H), gates (T,B,E) (the reference's gate_log, :298).
 * fp32-class accuracy (3xTF32 on the tensor cores); the (B,E,H) expert outputs stay on chip.  1 <= d <= 128, 1 <= E <= 8,
 * 1 <= H <= 1024 and 1 <= T <= 4 (CTR_ERR_UNSUPPORTED otherwise); B = 0 launches nothing.
 * workspace: 128-byte aligned, at least ctr_mmoe_workspace_bytes(0, d, E, H, T) bytes for the forward (the prepped
 * weights) and ctr_mmoe_workspace_bytes(B, d, E, H, T) for the backward (also the expert and gate-logit gradients,
 * (B, E*HP + 32) floats with HP = H rounded up to 32).  The backward takes the forward's gates and g_towers (T,B,H), and overwrites d_x (B,d),
 * d_w_experts (E,d,H), d_b_experts (E,H) and d_w_gates (T,d,E) (zeros at B = 0). */
int ctr_mmoe_workspace_bytes(int64_t B, int64_t d, int64_t E, int64_t H, int64_t T, int64_t* bytes);
int ctr_mmoe_fwd(const float* x, const float* w_experts, const float* b_experts, const float* w_gates, int64_t B, int64_t d,
                 int64_t E, int64_t H, int64_t T, float* towers, float* gates, void* workspace, int64_t workspace_bytes,
                 void* stream);
int ctr_mmoe_bwd(const float* x, const float* w_experts, const float* b_experts, const float* w_gates, const float* gates,
                 const float* g_towers, int64_t B, int64_t d, int64_t E, int64_t H, int64_t T, float* d_x,
                 float* d_w_experts, float* d_b_experts, float* d_w_gates, void* workspace, int64_t workspace_bytes,
                 void* stream);

/* ---- PLE extraction network and final gate layer ---------------------------------------------------------
 * Replaces extraction_network (PLE/extraction_network.py:4-85, extraction = 1) and the final experts and gates of
 * ple_model_fn (PLE/ple.py:185-226, extraction = 0).  T tasks with experts_per_task[t] = n_t >= 1 experts each (a host
 * array of T int64), S >= 1 shared experts, E = sum_t n_t + S experts in [task 0 .. task T-1, shared] order:
 *   h_e   = relu(x . w_e + b_e)           x (B,d); w_experts (E,d,H), b_experts (E,H)
 *   p_t   = softmax(x . gate_t)           over [task t's experts, shared experts]: n_t + S columns, no bias
 *   p_all = softmax(x . all_gate)         over all E experts (extraction = 1 only)
 *   w_gates (d, GC): the gate kernels concatenated by columns, gate_0 .. gate_{T-1} (then all_gate);
 *   GC = sum_t (n_t + S) (+ E).  gates (B, GC): the softmax probabilities, the same column layout.
 *   extraction = 0: out (T,B,H), out_t = sum_j p_t[j] h_(t, j);
 *   extraction = 1: out (B,H), the sum of the T task outputs and the all-gate output.
 * fp32-class accuracy (3xTF32 on the tensor cores); the (B,E,H) expert outputs stay on chip.  1 <= d <= 512,
 * 1 <= H <= 512, 1 <= T <= 4, E <= 64 and GC <= 160 (CTR_ERR_UNSUPPORTED otherwise); B = 0 launches nothing.
 * workspace: 128-byte aligned, at least ctr_ple_workspace_bytes(0, ...) bytes for the forward (the prepped weights) and
 * ctr_ple_workspace_bytes(B, ...) for the backward, which adds the expert and gate-logit gradients: (B, E*HP + GP)
 * floats with HP = H and GP = GC rounded up to 64 -- about 25.6 KB per sample at E = 25, H = 256.  The backward takes the
 * forward's gates and g_out (shaped as out), and overwrites d_x (B,d), d_w_experts (E,d,H), d_b_experts (E,H) and
 * d_w_gates (d,GC) (zeros at B = 0). */
int ctr_ple_workspace_bytes(int64_t B, int64_t d, int64_t H, int64_t T, const int64_t* experts_per_task, int64_t S,
                            int64_t extraction, int64_t* bytes);
int ctr_ple_fwd(const float* x, const float* w_experts, const float* b_experts, const float* w_gates, int64_t B, int64_t d,
                int64_t H, int64_t T, const int64_t* experts_per_task, int64_t S, int64_t extraction, float* out,
                float* gates, void* workspace, int64_t workspace_bytes, void* stream);
int ctr_ple_bwd(const float* x, const float* w_experts, const float* b_experts, const float* w_gates, const float* gates,
                const float* g_out, int64_t B, int64_t d, int64_t H, int64_t T, const int64_t* experts_per_task, int64_t S,
                int64_t extraction, float* d_x, float* d_w_experts, float* d_b_experts, float* d_w_gates, void* workspace,
                int64_t workspace_bytes, void* stream);

/* ---- Row MTL: multi-task loss balancing (uncertainty weighting, GradNorm, PCGrad) -------------------------
 * The reference sums its per-task losses (MMOE/mmoe.py:261-263, PLE/ple.py:251-254: tf.add_n); its README lists
 * "Uncertainty, GradNorm, PCGrad" as a to-do, so no reference code exists and these definitions are the contract.
 * T tasks, 1 <= T <= 8; B (samples) and P (shared-parameter floats) in 0..2^31-1; CTR_ERR_UNSUPPORTED naming the bound
 * otherwise.  L_t = mean_b sigmoid_ce(logit[t,b], label[t,b]) in TF's stable form (as ctr_sigmoid_ce).
 *   method 0, sum:         total = sum_t L_t                                   (the reference's add_n)
 *   method 1, weights:     total = sum_t w_t L_t                               (GradNorm's network loss; task_param = w)
 *   method 2, uncertainty: total = sum_t exp(-s_t) L_t + s_t / 2               (Kendall et al. 2018, eq. 10; task_param = s
 *                          = log sigma_t^2);  d total / d s_t = -exp(-s_t) L_t + 1/2
 * ctr_multitask_sigmoid_ce: logits, labels (T,B); task_param (T) (unused, may be NULL, for method 0).  Writes task_loss (T),
 * unweighted, and total_loss (1).  d_logits (T,B) (nullable) receives the UNWEIGHTED (sigmoid(x) - z) / B, so that it serves
 * the total (times 1, w_t or exp(-s_t)) and each L_t alone; d_task_param (T) (nullable) receives d total / d task_param
 * (L_t for method 1, zeros for method 0).  Deterministic: one cluster of 8 CTAs with a fixed partition and summation order
 * in float64, so the same inputs give the same bits.  B = 0 gives zero task losses.
 * Per-task gradients: grads holds T rows of P floats, row t = d L_t / d W over the shared parameters W (flattened), row
 * pitch ld >= P floats, any alignment.
 * ctr_multitask_gram: gram (T,T) float64 = grads . grads^T, one streaming pass over the T*P floats and a second one-CTA
 * pass over the per-CTA partials; deterministic.  workspace: at least ctr_multitask_gram_workspace_bytes(T, P) bytes,
 * 8-byte aligned.
 * ctr_pcgrad_combine (Yu et al. 2020, Algorithm 1): g_i' = g_i; for j in order (a permutation of 0..T-1, int32, device;
 * other entries are skipped), j != i: if g_i'.g_j < 0 then g_i' -= (g_i'.g_j / |g_j|^2) g_j; out (P) = sum_i g_i'.  Solved
 * in coefficient space from gram (C = I; dot = sum_k C_ik gram_kj; C_ij -= dot / gram_jj when dot < 0 and gram_jj > 0),
 * then out = sum_k (sum_i C_ik) g_k accumulated in float64.  coef (T, float64, nullable) receives sum_i C_ik.  A zero row
 * never triggers a projection; at T = 1 out equals the row bit for bit.
 * ctr_gradnorm_update (Chen et al. 2018, Algorithm 1), one small CTA in float64: n_t = sqrt(gram_tt) (gram of the
 * unweighted d L_t / d W), G_t = w_t n_t, Gbar = mean_t G_t, r_t = (L_t / L0_t) / mean_k (L_k / L0_k),
 * grad_loss (1) = sum_t |G_t - Gbar r_t^alpha| (the target is a constant), d_weights (T, nullable) = sign(G_t - Gbar
 * r_t^alpha) n_t with sign(0) = 0; then weights (T, in place) <- w - lr d_weights, renormalised to sum T.  No clamp: a large
 * lr can drive a weight negative.  initial_loss (L0) must be positive.  When every current loss is 0 (B = 0, or a batch
 * fitted exactly) r_t is undefined: weights are left unchanged, d_weights and grad_loss are 0. */
int ctr_multitask_sigmoid_ce(const float* logits, const float* labels, int64_t T, int64_t B, int method,
                             const float* task_param, float* task_loss, float* total_loss, float* d_logits,
                             float* d_task_param, void* stream);
int ctr_multitask_gram_workspace_bytes(int64_t T, int64_t P, int64_t* bytes);
int ctr_multitask_gram(const float* grads, int64_t T, int64_t P, int64_t ld, double* gram, void* workspace,
                       int64_t workspace_bytes, void* stream);
int ctr_pcgrad_combine(const float* grads, int64_t T, int64_t P, int64_t ld, const double* gram, const int32_t* order,
                       float* out, double* coef, void* stream);
int ctr_gradnorm_update(const double* gram, const float* task_loss, const float* initial_loss, int64_t T, float alpha,
                        float lr, float* weights, float* grad_loss, float* d_weights, void* stream);

/* ---- Row DIN-ATT: DIN attention unit -----------------------------------------------------------------
 * Replaces din_attention(query, keys, keys_length, is_softmax) (DIN/din_attention.py:17-43).
 * query (B,H); keys (B,T,H); keys_length int64 (B); dense layers f1_att (4H->64, relu), f2_att (64->32,
 * relu), f3_att (32->1): w1 (4H,64) b1 (64) w2 (64,32) b2 (32) w3 (32) b3 (1); out (B,H).
 * att_w (B,T): the final per-position weights (saved for backward), or NULL.
 * sched_scratch: device int32[B + 64] or NULL.  When given, a one-CTA pass orders the samples by descending keys_length and
 * the warps take them from a shared counter (longest-first list scheduling: a warp's cost is its samples' lengths); NULL =
 * static round-robin.  Same results either way (weight gradients are fp32-atomic sums in both). */
int ctr_din_attention_fwd(const float* query, const float* keys, const int64_t* keys_length,
                          const float* w1, const float* b1, const float* w2, const float* b2,
                          const float* w3, const float* b3, int64_t B, int64_t T, int64_t H, int is_softmax,
                          float* out, float* att_w, int32_t* sched_scratch, void* stream);
/* d_params: one flat fp32 buffer laid out [w1 | b1 | w2 | b2 | w3 | b3] (4H*64+64+64*32+32+32+1), overwritten.
 * att_w: the (B,T) weights saved by the forward, or NULL (they are then recomputed). */
int ctr_din_attention_bwd(const float* query, const float* keys, const int64_t* keys_length,
                          const float* w1, const float* b1, const float* w2, const float* b2,
                          const float* w3, const float* b3, const float* g_out, const float* att_w,
                          int64_t B, int64_t T, int64_t H, int is_softmax,
                          float* d_query, float* d_keys, float* d_params, int32_t* sched_scratch, void* stream);

/* ---- Row DIEN: interest extractor, attention and interest evolution ----------------------------------------
 * Replaces the seq_encoder block of dien_model_fn (DIEN/dien.py:198-229) with the cells of DIEN/custom_grucell.py:19-167 and
 * the loop of DIEN/rnn.py:443-798 (_rnn_step with skip_conditionals, :143-216):
 *   h_t  = GRUCell(nh) over seq_input (B,T,na) from a zero state, every position (dien.py:202-204);
 *   a    = softmax_t(h_t . (W_att e)), scores at t >= seq_length replaced by -2^32 + 1 (dien.py:206-218), e = target_input (B,na);
 *   s    = AGRU (cell_type 0, dien.py:223: any custom_gru_type other than "AUGRU") or AUGRU (cell_type 1) over h with the
 *          weights a, state copied through for t >= seq_length (dien.py:225-229);  final_state (B,nh) = s after step len-1
 *          (zero for len <= 0; len > T acts as T).  att_scores (B,T) = a, or NULL.
 * params: the nine variables packed in this order (floats):
 *   rnn/gru_cell/gates/kernel (na+nh, 2nh) | rnn/gru_cell/gates/bias (2nh) | rnn/gru_cell/candidate/kernel (na+nh, nh) |
 *   rnn/gru_cell/candidate/bias (nh) | attention_project_matrix (nh, na) | rnn/gates/kernel (2nh, 2nh) | rnn/gates/bias (2nh) |
 *   rnn/candidate/kernel (2nh, nh) | rnn/candidate/bias (nh)       (kernels: input rows first, then state rows).
 * workspace: ctr_dien_workspace_bytes() bytes; the forward keeps the states and weights the backward reads there, so the pair
 * must share one workspace.  The backward overwrites d_seq_input (B,T,na; exactly 0 at t >= len), d_target_input (B,na) and
 * d_params (packed like params; for AGRU the u half of rnn/gates/kernel and rnn/gates/bias gets exactly 0).
 * na <= 64, nh <= 64, T <= 128 (CTR_ERR_UNSUPPORTED otherwise). */
int ctr_dien_workspace_bytes(int64_t B, int64_t T, int64_t na, int64_t nh, int64_t* bytes);
int ctr_dien_fwd(const float* seq_input, const int64_t* seq_length, const float* target_input, const float* params, int64_t B,
                 int64_t T, int64_t na, int64_t nh, int cell_type, float* final_state, float* att_scores, void* workspace,
                 int64_t workspace_bytes, void* stream);
int ctr_dien_bwd(const float* seq_input, const int64_t* seq_length, const float* target_input, const float* params,
                 const float* g_final_state, int64_t B, int64_t T, int64_t na, int64_t nh, int cell_type, float* d_seq_input,
                 float* d_target_input, float* d_params, void* workspace, int64_t workspace_bytes, void* stream);

/* DIEN auxiliary loss (DIEN/dien.py:256-300, added to the loss at :316-317): next-behaviour supervision of the extractor
 * states h_t of ctr_dien_fwd.  With L = clamp(seq_length, 0, T), w_aux = aux_loss/aux_project_matrix W (na, nh),
 * neg_seq_input (B, (T-1)*T_neg, na) whose row t*T_neg + n is negative n of position t (the reshape at :279), and
 * q_t = W h_t (na):
 *   aux_loss = -(1/B) sum_b sum_{t < L-1} [ log sig(q_t . x_{t+1}) + sum_n log(1 - sig(q_t . neg_{t,n})) ]
 * -- the NEGATIVE of the reference's aux_loss (which, added to the loss as written, would be minimised toward -inf), in the
 * stable forms log sig(z) = -softplus(-z), log(1 - sig(z)) = -softplus(z).  Positions t >= L-1 are never computed.  The sum
 * is fixed-order (float64): the same inputs give the same bits.  B = 0 gives 0.
 * ctr_dien_aux_workspace_bytes(): the DIEN workspace plus B*(T-1) per-position terms; one such workspace serves ctr_dien_fwd,
 * ctr_dien_aux_fwd and ctr_dien_bwd_aux.  ctr_dien_aux_fwd reads the states ctr_dien_fwd left there, so it runs after it.
 * ctr_dien_bwd_aux: ctr_dien_bwd with the auxiliary loss's gradient added, given g_aux_loss, a DEVICE scalar (no host
 * synchronisation: the call is graph-capturable).  With s = g_aux/B, g+_t = s (sig(z+_t) - 1), g-_{t,n} = s sig(z-_{t,n}):
 * d_neg_seq_input (B, (T-1)*T_neg, na) is overwritten (row (t,n) = g-_{t,n} q_t, exactly 0 at t >= L-1); d_seq_input gets
 * g+_t q_t at row t+1 on top of ctr_dien_bwd's gradient; dL/dh_t gets W^T (g+_t x_{t+1} + sum_n g-_{t,n} neg_{t,n}) on top of the
 * attention and evolution terms; d_w_aux (na, nh) is overwritten with sum (that vector) (x) h_t.  With g_aux = 0 the outputs
 * of ctr_dien_bwd are reproduced bit for bit.  DIEN's bounds, and T_neg >= 1 with B*(T-1)*T_neg*na < 2^31
 * (CTR_ERR_UNSUPPORTED otherwise).  B = 0 zeroes aux_loss / d_params and d_w_aux and launches nothing else. */
int ctr_dien_aux_workspace_bytes(int64_t B, int64_t T, int64_t na, int64_t nh, int64_t T_neg, int64_t* bytes);
int ctr_dien_aux_fwd(const float* seq_input, const float* neg_seq_input, const int64_t* seq_length, const float* w_aux,
                     int64_t B, int64_t T, int64_t na, int64_t nh, int64_t T_neg, float* aux_loss, void* workspace,
                     int64_t workspace_bytes, void* stream);
int ctr_dien_bwd_aux(const float* seq_input, const float* neg_seq_input, const int64_t* seq_length, const float* target_input,
                     const float* params, const float* w_aux, const float* g_final_state, const float* g_aux_loss, int64_t B,
                     int64_t T, int64_t na, int64_t nh, int64_t T_neg, int cell_type, float* d_seq_input,
                     float* d_neg_seq_input, float* d_target_input, float* d_params, float* d_w_aux, void* workspace,
                     int64_t workspace_bytes, void* stream);

/* ---- Rows SENET / BILINEAR: FiBiNET ---------------------------------------------------------------------
 * senet(input, embedding_dim, reduction_ratio) (FiBiNET/senet.py:26-34): x (B,F,K); w1 (F,r); w2 (r,F). */
int ctr_senet_fwd(const float* x, const float* w1, const float* w2, int64_t B, int64_t F, int64_t K, int64_t r,
                  float* out, void* stream);
int ctr_senet_bwd(const float* x, const float* w1, const float* w2, const float* g_out,
                  int64_t B, int64_t F, int64_t K, int64_t r, float* dx, float* dw1, float* dw2, void* stream);
/* bilinear_interaction_layer(input, embedding_dim, type, name) (FiBiNET/bilinear_interaction_layer.py:21-40).
 * type: 0 'all' w (K,K); 1 'each' w (F-1,K,K); 2 'interaction' w (F(F-1)/2,K,K).
 * Pairs are itertools.combinations(range(F-1), 2) -- fields 0..F-2 only -- so out is (B, P, K) with
 * P = (F-1)(F-2)/2, exactly like the reference. */
int ctr_bilinear_fwd(const float* x, const float* w, int64_t B, int64_t F, int64_t K, int type,
                     float* out, void* stream);
int ctr_bilinear_bwd(const float* x, const float* w, const float* g_out, int64_t B, int64_t F, int64_t K, int type,
                     float* dx, float* dw, void* stream);
/* Tuning hook (process-wide, returns the previous mask; default 4).  Bit t (t = 0,1,2): type t runs the sample-batched
 * "tournament" kernels; otherwise 'all' / 'each' run the staged per-sample kernels and 'interaction' the round-1 kernels.
 * Bit 3: 'all' / 'each' use the round-1 CTA-per-sample kernels instead of the staged ones.  Bits 4..9: samples per tile of
 * the tournament kernels; bits 10..12: their weight columns per lane (1, 2, 4); 0 = chosen automatically.  The fast kernels
 * need K in {8,16,32} and 16-byte aligned arrays; other shapes always use the round-1 kernels.  Same results in every
 * setting; used by the parity tests (all forms) and tools/bench_layers.py for A/B timings. */
int ctr_bilinear_set_rr(int mask);

/* ---- SURVEY 8f.4: siblings of FM2 ------------------------------------------------------------------------------------------
 * NFM bi-interaction pooling (NFM/nfm.py:155-168): the fused gather of ctr_embed_fm2_fwd with a (B, D) output
 * bi[b,:] = 0.5 * ((sum_f e_f)^2 - sum_f e_f^2) instead of its sum over D; tile may be NULL.  Backward:
 * row_grads[b,f,:] = d_tile[b,f,:] (nullable) + d_bi[b,:] * (S[b,:] - e[b,f,:]). */
int ctr_embed_bi_fwd(const float* table, const int64_t* field_row_offset, const int64_t* ids, int64_t B, int64_t F, int64_t D,
                     float* tile, float* bi, void* stream);
int ctr_embed_bi_bwd(const float* tile, const float* d_tile, const float* d_bi, int64_t B, int64_t F, int64_t D,
                     float* row_grads, void* stream);

/* FLEN field-wise bi-interaction (FwBI; Chen et al., arXiv:1911.04690).  The reference tree has no FLEN code (its README
 * lists FLEN as a to-do), so this definition is the contract.  field_group: a HOST array of F int32, each in [0, M), read
 * before any launch (the call stays capturable in a CUDA graph).  With p_m = sum_{f: group[f]=m} e_f and
 * q_m = sum_{f: group[f]=m} e_f^2 (element-wise over D):
 *   h[b,:] = sum_{i<j} kernel_mf[pair(i,j)] p_i p_j + bias_mf + sum_m kernel_fm[m] (p_m^2 - q_m) + bias_fm        h (B,D)
 * pair(i,j): row-major strict upper triangle of M x M (FwFM's utils.py:67-82 order); kernel_mf (M(M-1)/2,), may be NULL
 * only when M == 1; kernel_fm (M,); bias_mf, bias_fm (D,).  A group with no field contributes zero; a singleton group's
 * p_m^2 - q_m is exactly 0.
 * ctr_embed_fwbi_fwd: the fused gather of ctr_embed_fm2_fwd (ids int64, or int32 with ids_are_int32 != 0, when
 * ids64_out (nullable) receives the widened ids; OOV / out-of-range ids give zero rows); tile (nullable) receives the rows.
 * ctr_fwbi_fwd: the same layer over a given (B,F,D) tile.
 * ctr_fwbi_bwd (both forms): row_grads[b,f,:] = d_tile[b,f,:] (nullable) + d_h[b,:] * (sum_{j != m} kernel_mf[pair(m,j)] p_j
 * + 2 kernel_fm[m] (p_m - e_f)) for f in group m -- the IndexedSlices values of the fused form, d_tile of the tile form;
 * overwrites d_kernel_mf (may be NULL only when M == 1), d_kernel_fm, d_bias_mf and d_bias_fm (both sum_b d_h[b,:]), zeros
 * at B = 0.  D a power of two in 4..128, 1 <= F <= 256, 1 <= M <= 8 (CTR_ERR_UNSUPPORTED otherwise); table, tile, d_tile,
 * h, d_h and row_grads 16-byte aligned, the weights float-aligned.  B = 0 launches nothing. */
int ctr_embed_fwbi_fwd(const float* table, const int64_t* field_row_offset, const void* ids, int ids_are_int32, int64_t B,
                       int64_t F, int64_t D, const int32_t* field_group, int64_t M, const float* kernel_mf,
                       const float* kernel_fm, const float* bias_mf, const float* bias_fm, float* tile, float* h,
                       int64_t* ids64_out, void* stream);
int ctr_fwbi_fwd(const float* tile, int64_t B, int64_t F, int64_t D, const int32_t* field_group, int64_t M,
                 const float* kernel_mf, const float* kernel_fm, const float* bias_mf, const float* bias_fm, float* h,
                 void* stream);
int ctr_fwbi_bwd(const float* tile, const float* d_tile, const float* d_h, int64_t B, int64_t F, int64_t D,
                 const int32_t* field_group, int64_t M, const float* kernel_mf, const float* kernel_fm, float* row_grads,
                 float* d_kernel_mf, float* d_kernel_fm, float* d_bias_mf, float* d_bias_fm, void* stream);

/* FwFM second-order logit (FwFM/fwfm.py:140-158): out[b] = sum_{i<j} r[pair(i,j)] * <tile[b,i,:], tile[b,j,:]>, r (F(F-1)/2,)
 * indexed like utils.py:67-82 (row-major strict upper triangle).  Backward: d_tile (B,F,K) and d_r (overwritten). */
int ctr_fwfm_fwd(const float* tile, const float* r, int64_t B, int64_t F, int64_t K, float* out, void* stream);
int ctr_fwfm_bwd(const float* tile, const float* r, const float* g, int64_t B, int64_t F, int64_t K, float* d_tile, float* d_r,
                 void* stream);

/* FFM second-order logit (FFM/ffm.py:128-160).  tile (B, F, F-1, K): the lookup of a table whose row for an id of field i is the
 * concatenation of its F-1 sub-embeddings, slot s facing field j = s+1 (s >= i) or s (s < i) -- i.e. the reference's
 * embedding_variables[i] of shape (F-1, |V_i|, K) stored id-major.  out[b] = sum_{i<j} <tile[b,i,j-1,:], tile[b,j,i,:]>.
 * Backward: d_tile[b,i,s,:] = g[b] * tile[b, partner(i,s), :] (overwritten). */
int ctr_ffm_fwd(const float* tile, int64_t B, int64_t F, int64_t K, float* out, void* stream);
int ctr_ffm_bwd(const float* tile, const float* g, int64_t B, int64_t F, int64_t K, float* d_tile, void* stream);

/* AFM attention pooling (AFM/afm.py:152-186): pairs (i<j) in the reference's order, a_p = h^T relu(W^T (e_i*e_j) + b),
 * softmax over the pair axis, pooled (B,K) = sum_p s_p (e_i*e_j).  w (K,T) row-major, b (T,), h (T,); score (B,P) optional
 * output.  K in {4,8,16,32} with K*ceil(T/32) <= 64.  Backward overwrites d_tile (B,F,K), d_w, d_b, d_h. */
int ctr_afm_fwd(const float* tile, const float* w, const float* b, const float* h, int64_t B, int64_t F, int64_t K, int64_t T,
                float* pooled, float* score, void* stream);
int ctr_afm_bwd(const float* tile, const float* w, const float* b, const float* h, const float* g_pooled, int64_t B, int64_t F,
                int64_t K, int64_t T, float* d_tile, float* d_w, float* d_b, float* d_h, void* stream);

/* BST transformer block (BST/transformer_layer.py:6-79): queries/keys/values (B,T,d), keys_length (B,) int64 (mask t >= length,
 * applied along the QUERY axis as the reference does, float32 collapse included), heads >= 1 (each projecting to d),
 * position embedding rows [0,T) of a (max_length,d) table added to queries and keys.  params packed as
 *   position_embedding (max_length,d) | w_q (H,d,d) | w_k | w_v | w_o (H*d,d) | LayerNorm beta,gamma (d,d) |
 *   dense kernel (d,d), bias (d) | LayerNorm_1 beta,gamma        = ctr_bst_param_count(d, heads, max_length) floats.
 * out (B,T,d).  Backward recomputes the forward; d_queries/d_keys/d_values (B,T,d) and d_params (same packing) are
 * overwritten.  One CTA per sample: d in {4,8,16,32,64}, T <= 128, heads <= 16 and a shared-memory footprint <= 220 KB, else -2. */
int64_t ctr_bst_param_count(int64_t d, int64_t heads, int64_t max_length);
int ctr_bst_transformer_fwd(const float* queries, const float* keys, const float* values, const int64_t* keys_length,
                            const float* params, int64_t B, int64_t T, int64_t d, int64_t heads, int64_t max_length,
                            int use_position_embedding, float* out, void* stream);
int ctr_bst_transformer_bwd(const float* queries, const float* keys, const float* values, const int64_t* keys_length,
                            const float* params, const float* g_out, int64_t B, int64_t T, int64_t d, int64_t heads,
                            int64_t max_length, int use_position_embedding, float* d_queries, float* d_keys, float* d_values,
                            float* d_params, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CTR_B200_H_ */

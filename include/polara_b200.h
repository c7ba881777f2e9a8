/*
 * polara_b200 -- C-ABI of the H100-native factorization-and-scoring engine.
 *
 * The reference (evfro/polara, pure Python) has NO FFI of its own: its hot path
 * bottoms out in scipy/numpy/numba calls.  Each entry point below replaces one
 * of those call sites (cited per function; paths relative to the reference
 * checkout) and is what a ctypes binding on the reference side would bind --
 * see INTEGRATION.md for that binding.
 *
 * Conventions
 *   - every function returns an int status: 0 = OK, PB200_E* otherwise;
 *     pb200_last_error(ctx) gives the message.
 *   - all array arguments are DEVICE pointers (cudaMalloc'ed by the caller, e.g.
 *     torch tensors' data_ptr()) unless the name ends in _host.
 *   - work is enqueued on the context's stream; nothing synchronises unless noted.
 *   - CSR: indptr int64 [n_rows+1], indices int32 [nnz] (sorted within a row),
 *     values float32 [nnz].  Dense matrices are row-major float32 with an explicit
 *     leading dimension (ld, in elements).
 *   - sm_90a (H100) only.  No CPU fallback exists.
 */
#ifndef POLARA_B200_H
#define POLARA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PB200_OK 0
#define PB200_EINVAL 1   /* -> ValueError   */
#define PB200_ENOMEM 2   /* -> MemoryError  */
#define PB200_ECUDA 3    /* -> RuntimeError */
#define PB200_ENOTIMPL 4 /* -> NotImplementedError */

typedef struct pb200_ctx pb200_ctx;

/* candidate list entry produced by the scoring kernels */
typedef struct { float score; int32_t id; } pb200_cand;

int pb200_version(void);

/* stream: a cudaStream_t (e.g. torch.cuda.current_stream().cuda_stream) or NULL
 * for the legacy default stream. */
int pb200_ctx_create(int device, void* stream, pb200_ctx** out);
int pb200_ctx_destroy(pb200_ctx* ctx);
/* later work is enqueued on `stream` (the caller orders it against earlier work on the previous stream). */
int pb200_ctx_set_stream(pb200_ctx* ctx, void* stream);
const char* pb200_last_error(pb200_ctx* ctx);
int pb200_ctx_sync(pb200_ctx* ctx);
/* development aid: prints the diagnostics a timed-out (trapped) kernel left in pinned host memory to stderr */
int pb200_debug_dump(pb200_ctx* ctx);
/* which scoring kernel pb200_score_topk uses: 0 = exact SIMT fp32 kernel,
 * 1 = tc (bf16 wgmma tensor-core filter + exact fp32 rescoring; same results). */
int pb200_set_score_kernel(pb200_ctx* ctx, int kind);
/* 1 (default): a user tile's sweep over the norm-ordered items stops at the first position where
 * ||e_u|| * ||v_pos|| (Cauchy-Schwarz) can no longer reach the user's seeded k-th best score -- results are unchanged
 * (the skipped pairs cannot enter a top-k list); 0: every (user, item) pair goes through the tensor-core filter. */
int pb200_set_prune(pb200_ctx* ctx, int on);
/* counters of the last scoring call (host array of 8 uint64):
 *  [0] kernels launched  [1] candidates rescored  [2] item tiles  [3] user tiles
 *  [4] duration of the last fused scoring kernel in microseconds (CUDA events on the
 *      context stream; synchronises)
 *  [5] (user tile x item tile) products the tensor-core sweep executed so far (cumulative over calls)
 *  [6] the same count had no sweep been cut short by the norm bound (pb200_set_prune)
 *  [7] non-zero: a kernel gave up on a barrier (diagnostic code) */
int pb200_get_stats(pb200_ctx* ctx, uint64_t* out8_host);

/* Row-sharded build (SURVEY.md 8e "Partitioning - build": users split across GPUs, one process per GPU).
 * The hook must replace the `count` elements at `dev_ptr` by their sum over all shards, ordered after prior work on
 * the context stream and before later work on it (e.g. ncclAllReduce on that stream, or torch.distributed.all_reduce
 * with the context stream current).  While a hook is installed pb200_rsvd and pb200_rescale treat their CSR
 * arguments as this rank's ROW BLOCK of the matrix: Gram matrices of user-side panels (f64, ell*ell), the
 * item-side panel A^T W (f32, n_cols*ell) and the column counts of pb200_rescale (i32, n_cols) go through it.
 * Every rank must make the same calls in the same order.  fn == NULL removes the hook.  Returns 0 on success. */
#define PB200_F32 0
#define PB200_F64 1
#define PB200_I32 2
typedef int (*pb200_reduce_fn)(void* user, void* dev_ptr, int64_t count, int dtype);
int pb200_set_reduce_hook(pb200_ctx* ctx, pb200_reduce_fn fn, void* user);

/* Item-sharded scoring (SURVEY.md 8e "Partitioning - scoring": every rank scores ALL users against its own item shard).
 * Between its probe pass and its sweep the tensor-core scoring path holds, per user, a lower bound of the user's final k-th
 * best score (the k-th best exact score among the shard's largest-norm unseen items).  A bound found on ANY shard holds for
 * the merged result, so the hook, called once per pb200_score_topk / pb200_score_topk_cands that the tensor-core path takes
 * (not by the CUDA-core kernel: pb200_set_score_kernel(0) or ranks above 509, which keep no such bounds; the choice depends
 * on the rank and the device only, so all ranks of a job agree) as fn(user, bounds, n_users, PB200_F32), must replace the
 * n_users floats at `bounds` by their elementwise MAXIMUM over all ranks (same ordering rules as the reduce hook; every rank
 * scores the same users in the same call order).  Shards whose items cannot reach another
 * shard's bound then stop their sweep early instead of producing candidates the merge would drop: results are unchanged.
 * Remove the hook (fn == NULL) before scoring calls that are not part of such a sharded job.  No reference counterpart. */
int pb200_set_bound_hook(pb200_ctx* ctx, pb200_reduce_fn fn, void* user);

/* A CSR matrix resident in HBM, optionally stored PANEL-MAJOR (pb200_csr_block_columns): the columns are cut into
 * n_panels panels of panel_cols columns, the nnz of panel 0 come first (rows in order, columns sorted), then panel 1, ...;
 * indptr has n_panels * n_rows + 1 entries (virtual row = panel * n_rows + row), indices are GLOBAL column ids.
 * n_panels == 1 is a plain CSR.  panel_ptr_host (HOST memory, n_panels + 1 entries, may be NULL when n_panels == 1)
 * holds the nnz offset at which each panel starts: the launch grids are sized from it without a device round trip. */
typedef struct {
    int64_t n_rows, n_cols, nnz;
    const int64_t* indptr;
    const int32_t* indices;
    const float* values;
    int32_t n_panels;
    int64_t panel_cols;
    const int64_t* panel_ptr_host;
} pb200_csr_view;

/* which SpMM kernel runs (all deterministic, same results up to the summation order of rows that straddle windows):
 *   3 (default) nnz windows per warp + 128-bit register gathers (a lane owns four columns; half a warp per nnz up to 64
 *               columns, a full warp up to 128): work split by nnz, carried row pieces added in order;
 *   4           the same with 32-bit gathers (a lane owns one column per 32-column group; also taken for operands that
 *               are not 16-byte aligned);
 *   1 / 2       dense rows of X staged in shared memory by cp.async.bulk (one UBLKCP per row) / by 16-byte cp.async --
 *               the per-row copy issue limits them; operands that are not
 *               16-byte aligned fall back to 0;
 *   0           row-owned register gathers (round-1 kernel). */
int pb200_set_spmm_kernel(pb200_ctx* ctx, int kind);

/* Y[n_rows x ell] = A * X ; replaces csr_matrix.dot(ndarray) at
 * polara/recommender/models.py:860 (P.dot(V)) and the A x / A^T x products inside
 * scipy svds (models.py:844).  X is read up to column ell only (ldx >= ell); Y is written in whole groups of 32
 * columns, zero beyond ell (ldy >= ell rounded up to 32). */
int pb200_spmm(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
               const int64_t* indptr, const int32_t* indices, const float* values,
               const float* X, int64_t ldx, float* Y, int64_t ldy, int ell);

/* same product for a matrix view (plain or panel-major); with panels Y accumulates in panel order (deterministic). */
int pb200_spmm_csr(pb200_ctx* ctx, const pb200_csr_view* a, const float* X, int64_t ldx, float* Y, int64_t ldy, int ell);

/* Panel-major copy of a CSR matrix (see pb200_csr_view): a format conversion done once per build() so that the slice
 * of the dense operand one panel gathers from (panel_cols rows of X) stays resident in the 50 MB L2 while the nnz
 * stream through.  b_indptr [n_panels * n_rows + 1], b_indices/b_values [nnz] device; panel_ptr_host [n_panels + 1] HOST.
 * n_panels must equal ceil(n_cols / panel_cols).  Synchronises the stream (the panel offsets are returned to the host). */
int pb200_csr_block_columns(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                            const int64_t* indptr, const int32_t* indices, const float* values,
                            int64_t panel_cols, int n_panels,
                            int64_t* b_indptr, int32_t* b_indices, float* b_values, int64_t* panel_ptr_host);

/* Device-side ingest of the triplets a Polara data model hands to a model: RecommenderData.to_coo (data.py:794-817:
 * idx intp [nnz x 2], val) and test_to_coo (data.py:835-862: user, item, feedback arrays) -> CSR with duplicates summed
 * and columns sorted; replaces coo_matrix(...).tocsr() at models.py:169-174 and csr_matrix((fdbk,(user,item))) at
 * models.py:208-210.  rows/cols: device int64 with element strides (idx[:, 0] / idx[:, 1] of a row-major [nnz x 2] array
 * have stride 2); vals: device float32/float64 (val_dtype PB200_F32 / PB200_F64) or NULL = all ones;
 * drop_zeros != 0 removes zero-valued triplets first (get_test_matrix, models.py:197-201);
 * require_sorted_rows != 0 makes decreasing row ids an error (PB200_EINVAL) -- the reference asserts that test triplets
 * are sorted by user (models.py:246).
 * Outputs: indptr_out [n_rows + 1], indices_out / values_out with room for nnz entries; *nnz_out_host (HOST) = entries
 * written.  Input already strictly increasing in (row, col) is converted without sorting.  Synchronises the stream. */
int pb200_coo_to_csr(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                     const int64_t* rows, int64_t row_stride, const int64_t* cols, int64_t col_stride,
                     const void* vals, int val_dtype, int drop_zeros, int require_sorted_rows,
                     int64_t* indptr_out, int32_t* indices_out, float* values_out, int64_t* nnz_out_host);

/* pb200_coo_to_csr (same CSR, same bits), plus what rewriting the values later needs: perm_out int64 [nnz] = the
 * stable sort's permutation (sorted position -> input position; the identity when the input was strictly increasing)
 * and run_ptr_out int64 [nnz_out + 1] = where each stored entry's run of summed duplicates starts in sorted order
 * (run_ptr_out[nnz_out] = the end of the last run).  Sizes the outputs for the nnz input entries. */
int pb200_coo_to_csr_runs(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                          const int64_t* rows, int64_t row_stride, const int64_t* cols, int64_t col_stride,
                          const void* vals, int val_dtype, int drop_zeros, int require_sorted_rows,
                          int64_t* indptr_out, int32_t* indices_out, float* values_out, int64_t* nnz_out_host,
                          int64_t* perm_out, int64_t* run_ptr_out);

/* values_out[o] (float32, n_unique stored entries) = the sum over entry o's run of table[levels[perm[j]]] (table
 * float32 [n_levels], levels int64 [nnz] per input triplet), in the order and at the precision pb200_coo_to_csr sums
 * float32 values: the CSR of pb200_coo_to_csr_runs then holds the same bits as a fresh pb200_coo_to_csr of the float32
 * weights table[levels].  CoFFee's test matrix at another multilinear rank (models.py:1312-1315).  Synchronises the
 * stream; a level outside [0, n_levels) is PB200_EINVAL. */
int pb200_csr_values_from_table(pb200_ctx* ctx, int64_t n_unique, const int64_t* run_ptr, const int64_t* perm,
                                const int64_t* levels, const float* table, int64_t n_levels, float* values_out);

/* x[i] += delta for i < count (device int64): re-bases the row pointers / user ids of a chunk of a larger matrix. */
int pb200_shift_i64(pb200_ctx* ctx, int64_t* x, int64_t count, int64_t delta);

/* CSR of A^T (= CSC of A), rows sorted; scipy's coo->csr/csc conversion at
 * models.py:169-174 plays this role on the CPU. */
int pb200_csr_transpose(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                        const int64_t* indptr, const int32_t* indices, const float* values,
                        int64_t* t_indptr, int32_t* t_indices, float* t_values);

/* In place: values <- D_r^(row_scaling-1) A D_c^(col_scaling-1), D = diag(sqrt(nnz count))
 * ; polara/preprocessing/matrices.py:71-93 (binary=True) as called from
 * ScaledMatrixMixin.get_training_matrix, models.py:891-895. */
int pb200_rescale(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                  const int64_t* indptr, const int32_t* indices, float* values,
                  double row_scaling, double col_scaling);

/* Truncated SVD by randomized subspace iteration; replaces
 * scipy.sparse.linalg.svds at models.py:844.  Needs both A (CSR) and A^T (CSR).
 *   V_out [n_cols x ldv]  right singular vectors, column j pairs with sigma_out[j]
 *   sigma_out [rank] float64, descending (models.py:846-855 ordering)
 *   U_out [n_rows x ldu] or NULL
 *   ell: subspace width (multiple of 32, > rank); max_iters: power iterations;
 *   tol: stop when the leading `rank` Ritz values move less than tol (relative)
 *   iters_done_host: host int, may be NULL. Synchronises the stream. */
int pb200_rsvd(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
               const int64_t* indptr, const int32_t* indices, const float* values,
               const int64_t* t_indptr, const int32_t* t_indices, const float* t_values,
               int rank, int ell, int max_iters, double tol, uint64_t seed,
               float* V_out, int64_t ldv, double* sigma_out, float* U_out, int64_t ldu,
               int* iters_done_host);

/* Same factorisation for matrix views (A and A^T may be panel-major).  info_host (HOST, 8 doubles, may be NULL):
 *   [0] subspace iterations done   [1] largest relative change of the leading `rank` Ritz values in the last iteration
 *   [2] upper bound of sin(largest principal angle) between the leading-`rank` right subspaces of the last two iterates
 *   [3] 1 if both fell below tol / vec_tol before max_iters, else 0 (the caller should warn: the factors are the best
 *       subspace found, not a converged one)
 * vec_tol <= 0 disables the subspace test. */
int pb200_rsvd_csr(pb200_ctx* ctx, const pb200_csr_view* A, const pb200_csr_view* At,
                   int rank, int ell, int max_iters, double tol, double vec_tol, uint64_t seed,
                   float* V_out, int64_t ldv, double* sigma_out, float* U_out, int64_t ldu, double* info_host);

/* The same factorisation of the matrix-free operator M = K_u^T A K_i (HybridSVD, hybrid/models.py:368-384): every
 * product of the subspace iteration and of the Rayleigh-Ritz step is the chain
 *   M X = K_u^T (A (K_i X))        M^T W = K_i^T (A^T (K_u W))
 * of SpMMs, so V_out / sigma_out / U_out are the right vectors, singular values and left vectors of M.  Each factor is a
 * pair of views (K, K^T), plain or panel-major; a NULL pair is the identity on that side (both NULL = pb200_rsvd_csr).
 * K_i, K_i^T are n_cols x n_cols and K_u, K_u^T n_rows x n_rows (A is n_rows x n_cols), else PB200_EINVAL.  Factors
 * under a reduce hook return PB200_ENOTIMPL: a user factor mixes rows of different shards.  Scratch: two more panels,
 * [n_cols x ell] and [n_rows x ell], when a factor is given. */
int pb200_rsvd_factored(pb200_ctx* ctx, const pb200_csr_view* A, const pb200_csr_view* At,
                        const pb200_csr_view* Ki, const pb200_csr_view* Kit,
                        const pb200_csr_view* Ku, const pb200_csr_view* Kut,
                        int rank, int ell, int max_iters, double tol, double vec_tol, uint64_t seed,
                        float* V_out, int64_t ldv, double* sigma_out, float* U_out, int64_t ldu, double* info_host);

/* Thin SVD pieces of a dense tall matrix M [n x c]: leading `rank` singular values
 * (sigma_out, float64, descending), left vectors U_out [n x ldu] and, if not NULL,
 * right vectors Vt_out [rank x c] (row-major).  Replaces svds() on the dense HOOI
 * unfoldings, polara/lib/tensor.py:71,75,79.  While a reduce hook is installed (pb200_set_reduce_hook) M is this rank's
 * block of ROWS: the c x c Gram matrix is summed over the ranks, sigma / Vt are global, U_out holds the rank's own rows
 * (the mode-0 step of a HOOI whose nnz are sharded by user). */
int pb200_tall_svd(pb200_ctx* ctx, const float* M, int64_t n, int c, int64_t ldm, int rank,
                   double* sigma_out, float* U_out, int64_t ldu, float* Vt_out);

/* Fused scores = E V^T  ->  seen-item masking -> per-row top-k; full score rows
 * never reach HBM.  Replaces the chain slice_recommendations (models.py:857-861,
 * the dgemm) -> downvote_seen_items (models.py:494-519) -> get_topk_elements
 * (models.py:522-564).
 *   E [m x lde] user embeddings (P V), V [n x ldv] item factors, r = rank
 *   seen_indptr/seen_indices: CSR of seen items per user (sorted, unique per row; ids in
 *       the OUTPUT id space, i.e. local item id + item_offset), NULL/NULL = filter_seen False
 *   out_ids int64 [m x k] (+ item_offset), out_scores float32 [m x k] or NULL.
 * Order: unseen items by (score desc, id asc); if fewer than k unseen items exist
 * the seen ones follow by (score desc, id asc) -- the order models.py:517-519 yields. */
int pb200_score_topk(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv,
                     int64_t m, int64_t n, int r,
                     const int64_t* seen_indptr, const int32_t* seen_indices,
                     int k, int64_t item_offset, int64_t* out_ids, float* out_scores);

/* Same, but stops at the per-row candidate list of THIS item shard:
 * out_cands [m x k] sorted, ids global (+item_offset), empty slots id=-1/score=-inf.
 * Used for item-factor sharding across GPUs. */
int pb200_score_topk_cands(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv,
                           int64_t m, int64_t n, int r,
                           const int64_t* seen_indptr, const int32_t* seen_indices,
                           int k, int64_t item_offset, pb200_cand* out_cands);

/* count empty entries {score = -inf, id = -1}: the padding rows of a candidate block that is exchanged between GPUs. */
int pb200_fill_empty_cands(pb200_ctx* ctx, pb200_cand* cands, int64_t count);

/* Merge `parts` sorted candidate lists per row: in [parts][m][k] -> ids/scores [m x k]. */
int pb200_merge_cands(pb200_ctx* ctx, const pb200_cand* in, int parts, int64_t m, int k,
                      int64_t* out_ids, float* out_scores);

/* Same merge on the rank that OWNS the rows after the exchange of an item-sharded job, completed with the reference's
 * seen-item fill-up (models.py:517-519): rows with fewer than k unseen candidates over all shards continue with their
 * seen items by (score desc, id asc), scored exactly from E [m x lde] (these rows' embeddings) and the WHOLE V [n x ldv].
 * in: parts lists of k entries per row, list p of row u at in[p * part_stride + u * k]; seen ids are global. */
int pb200_merge_cands_fill(pb200_ctx* ctx, const pb200_cand* in, int parts, int64_t part_stride, int64_t m, int k,
                           const float* E, int64_t lde, const float* V, int64_t ldv, int r, int64_t n,
                           const int64_t* seen_indptr, const int32_t* seen_indices,
                           int64_t* out_ids, float* out_scores);

/* out[a] = E[user_idx[a], :r] . V[item_idx[a], :r] for `count` (user, item) pairs (device int64 index arrays): the scores
 * of holdout items and of sampled unseen items in the sampled evaluation protocol -- inner_product_at
 * (polara/lib/sparse.py:58-72) as used by RandomSampleEvaluationSVDMixin (models.py:1095-1183).  Out-of-range indices
 * yield NaN.  The scores are the same canonical fp32 values the fused kernel ranks by. */
int pb200_gather_dot(pb200_ctx* ctx, const float* E, int64_t lde, int64_t m, const float* V, int64_t ldv, int64_t n,
                     int r, const int64_t* user_idx, const int64_t* item_idx, int64_t count, float* out);

/* On-the-fly sample of unseen items, the draw of the reference's sampled evaluation when no unseen interactions were
 * set (RandomSampleEvaluationSVDMixin.compute_random_item_scores_gen, models.py:1137-1156); replaces sample_row_wise
 * (polara/lib/sampler.py:96-111) and the draw inside mf_random_item_scoring (sampler.py:73-93), bit for bit: per user
 * numba's random.seed(seeds_u32[u]) (MT19937 init_genrand), prime_sampler_state over the exclusion list, then n_samples
 * draws randrange(remaining) through the position map.
 *   excl_indptr int64 [m+1], excl_indices int32: the exclusion list of each user.  EXCEPTION to the CSR convention
 *       above: the lists are ORDERED, NOT NECESSARILY SORTED, and are read in the given order (priming places the
 *       excluded items in list order, so a permuted list draws differently).  The reference forms them as scipy's
 *       profile + holdout sum (models.py:1145-1148), whose row order is scipy's when a holdout row is unsorted.
 *   seeds_u32 uint32 [m] (np.random.SeedSequence(data.seed).generate_state(m), models.py:1151)
 *   out_items int64 [m x ld_out]: the first n_samples columns of each row are written, nothing else (so the ids can be
 *       placed right after the h holdout columns of an index block).
 * PB200_EINVAL if a user has fewer than n_samples items left (the reference's randrange raises "empty range") or an
 * exclusion id lies outside [0, n_items).  Synchronises the stream (the check's verdict is read back). */
int pb200_sample_unseen(pb200_ctx* ctx, int64_t m, int64_t n_items, const int64_t* excl_indptr, const int32_t* excl_indices,
                        const uint32_t* seeds_u32, int n_samples, int64_t* out_items, int64_t ld_out);

/* The sampled evaluation fused: per user the draw of pb200_sample_unseen, the scores of the h holdout items
 * (holdout_items int64 [m x h]) and of the n_samples drawn items -- the canonical fp32 chain of pb200_gather_dot, bit
 * identical, NaN for holdout ids out of range, which never enter a list -- and the top-k POSITIONS in the row
 * [holdout | sampled] by (score desc, position asc): models.py:1158-1183 (compute_holdout_scores, mf_random_item_scoring,
 * np.apply_along_axis(topsort)).  No [m x (h + n_samples)] score or index block is formed.  out_pos int64 [m x k] (-1 pads
 * a row with fewer than k scorable entries), out_scores float32 [m x k] or NULL.  1 <= k <= h + n_samples.  Errors and
 * synchronisation as pb200_sample_unseen. */
int pb200_sampled_topk(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv, int64_t m, int64_t n,
                       int r, const int64_t* holdout_items, int h, const int64_t* excl_indptr, const int32_t* excl_indices,
                       const uint32_t* seeds_u32, int n_samples, int k, int64_t* out_pos, float* out_scores);

/* pb200_sampled_topk at several truncated ranks of one factor pair in one pass: the rank sweep of find_optimal_svd_rank
 * (evaluation/pipelines.py:81-116, truncation models.py:819-832) under the sampled protocol.  Each user is drawn once;
 * each drawn (and holdout) item's fp32 chain is continued from ranks[j-1] to ranks[j] and offered to list j, so each V
 * row is read once, up to the largest rank.  ranks_host: host array of n_ranks ints, strictly ascending,
 * 1 <= ranks[0], ranks[n_ranks-1] <= min(lde, ldv), 1 <= n_ranks <= 64.  out_pos int64 [n_ranks x m x k], rank-major
 * (block j has the layout of pb200_sampled_topk's output), out_scores float32 of the same layout or NULL.  For every j,
 * block j is bit-equal to pb200_sampled_topk(E, lde, V, ldv, m, n, ranks[j], ...) on the same E and V.  Errors and
 * synchronisation as pb200_sampled_topk, plus PB200_EINVAL for a rank list that is empty, too long, not strictly
 * ascending, below 1 or above lde / ldv. */
int pb200_sampled_topk_ranks(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv, int64_t m, int64_t n,
                             const int* ranks_host, int n_ranks, const int64_t* holdout_items, int h,
                             const int64_t* excl_indptr, const int32_t* excl_indices, const uint32_t* seeds_u32,
                             int n_samples, int k, int64_t* out_pos, float* out_scores);

/* Position-map placement of the two sampler entries: a user whose map (2 * |exclusion| + n_samples entries at most, at a
 * load factor <= 2/3) fits in `slots` 8-byte slots runs with the map in shared memory, the others with it in global
 * memory.  0..6144, default 3072; 0 puts every user on the global-memory path.  Results do not depend on it. */
int pb200_set_sampler_map_slots(pb200_ctx* ctx, int slots);
/* the last sampler call (host array of 4 uint64): [0] users on the shared-memory map path, [1] users on the global-memory
 * map path, [2] map slots per warp on the global path, [3] kernels launched. */
int pb200_sampler_stats(pb200_ctx* ctx, uint64_t* out4_host);

/* Dense scores S [m x lds] = E V^T for a handful of users (the single-user path of
 * models.py:277-293 expects a dense score row). */
int pb200_score_dense(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv,
                      int64_t m, int64_t n, int r, float* S, int64_t lds);

/* Top-k of a caller's dense score block S [m x lds] (float32 / float64 by `dtype` = PB200_F32 / PB200_F64), for scores
 * that did not come from our factors: RecommenderModel.get_topk_elements, dense branch (models.py:561-563; topsort
 * 488-491).  With a seen CSR (int64 indptr [m+1], int32 sorted ids) the seen-item handling is fused in: unseen items by
 * (score desc, id asc), then -- if fewer than k are unseen -- the seen ones in the same order, i.e. what
 * downvote_seen_items (models.py:510-519) followed by get_topk_elements yields.  out_ids int64 [m x k]; out_scores
 * [m x k] in the input dtype or NULL.  k > n is an error (np.argpartition raises there). */
int pb200_topk_dense(pb200_ctx* ctx, const void* S, int dtype, int64_t lds, int64_t m, int64_t n,
                     const int64_t* seen_indptr, const int32_t* seen_indices, int k, int64_t* out_ids, void* out_scores);

/* In place on a dense score block: S[row, col] <- min(S) - (max(S at the seen pairs) - S[row, col]) - 1 for the nnz seen
 * pairs (rows / cols: device int64) -- RecommenderModel.downvote_seen_items, dense branch (models.py:510-519):
 * order-preserving push below the block minimum. */
int pb200_downvote_dense(pb200_ctx* ctx, void* S, int dtype, int64_t lds, int64_t m, int64_t n,
                         const int64_t* rows, const int64_t* cols, int64_t nnz);

/* Item-to-item model (CooccurrenceModel, models.py:693-725).
 * pb200_cooc_build: S = A^T A with a zero diagonal (models.py:702-709) as a DENSE fp64 matrix S [n x lds], n = a->n_cols.
 *   `a` is the training CSR split into column panels of at most PB200_COOC_MAX_PANEL_BYTES / 8 columns
 *   (pb200_csr_block_columns; one panel when it is narrow enough), `at` the plain CSR of A^T (pb200_csr_transpose).
 *   implicit != 0 takes sign(a_ui) for every value (models.py:699-701).  Every entry is summed over the users in
 *   ascending order; fp32 products are exact in fp64, so integer-valued data gives S exactly (and exactly symmetric). */
#define PB200_COOC_MAX_PANEL_BYTES 196608
int pb200_cooc_build(pb200_ctx* ctx, const pb200_csr_view* a, const pb200_csr_view* at, int implicit, double* S,
                     int64_t lds);
/* pb200_i2i_topk: for each of the m test users (CSR p_*, the test matrix of get_test_matrix, models.py:180-211)
 * s_u = sum_i p_ui S[i, :] in fp64 with i ascending, a rounded product then a rounded sum (scipy's csr_matmat order;
 * implicit != 0 takes sign(p_ui)), and
 *   out_nnz    int64 [m]      |{j : s_uj != 0}| over all items, seen ones included;
 *   out_dense  int64 [m x k]  the dense-chunk rule (toarray + downvote_seen_items + topsort, models.py:510-519, 561-563):
 *                             unseen items by (score desc, id asc), zero scores included, then the seen ones in the same
 *                             order; without a seen CSR every item by (score desc, id asc);
 *   out_sparse int64 [m x k]  the sparse-chunk rule (models.py:524-560): the items with s != 0 by (score desc, id asc),
 *                             seen ones included, then -1 up to k.  downvote_seen_items' sparse branch (models.py:
 *                             501-509) has no effect on the caller's block: `recs -= seen_recs` rebinds a local name,
 *                             scipy's sparse matrices having no in-place subtraction;
 *   out_scores fp64 [m x k]   the scores of out_dense, or NULL.
 * seen_*: int64 indptr [m+1] / sorted int32 ids of the seen items, or both NULL.  1 <= k <= n.  No [m x n] block is
 * formed and each S row of a user is read once. */
int pb200_i2i_topk(pb200_ctx* ctx, const double* S, int64_t lds, int64_t n, int64_t m, const int64_t* p_indptr,
                   const int32_t* p_indices, const float* p_values, const int64_t* seen_indptr,
                   const int32_t* seen_indices, int implicit, int k, int64_t* out_nnz, int64_t* out_dense,
                   int64_t* out_sparse, double* out_scores);

/* Sparse storage of the item-to-item matrix, for catalogues whose dense S does not fit.
 * pb200_cooc_build_csr: the S of pb200_cooc_build as an fp64 CSR [n x n]: rows with ascending column ids, no diagonal
 *   and no entry that sums to exactly 0 (eliminate_zeros); every stored entry has the bits of the dense build's entry.
 *   `a` is the plain training CSR (one panel), `at` the plain CSR of A^T.  Two calls with the same a, at and implicit:
 *     fill == 0  counts the rows: indptr (device int64 [n+1]) gets the row offsets, *nnz (HOST) the total, so the
 *                caller can check the memory before allocating the rows;
 *     fill != 0  writes the rows (device int32 / fp64 [*nnz]) at those offsets; *nnz is the count of the first call
 *                (0: nothing to write, indices / values may be NULL).
 *   acc_rows: at most this many rows of n doubles of global scratch for the item rows whose work exceeds a
 *   shared-memory table (at least 1; each CTA of that path owns one; only as many as there are such rows are taken). */
int pb200_cooc_build_csr(pb200_ctx* ctx, const pb200_csr_view* a, const pb200_csr_view* at, int implicit, int acc_rows,
                         int fill, int64_t* indptr, int32_t* indices, double* values, int64_t* nnz);
/* pb200_i2i_topk_csr: pb200_i2i_topk with S given as an fp64 CSR [n x n] (s_indptr int64 [n+1], s_indices int32 sorted,
 *   s_values fp64), with the same outputs, bit-equal to pb200_i2i_topk on the dense form of the same S.  acc_rows: at
 *   most this many rows of n doubles of global scratch for the users whose work (the nonzeros of their S rows) exceeds
 *   a shared-memory table (at least 1; each warp of that path owns one; only as many as there are such users are
 *   taken).  Scratch besides: m * 2k * 16 + 24 m bytes.  No [m x n] block is formed. */
int pb200_i2i_topk_csr(pb200_ctx* ctx, int64_t n, const int64_t* s_indptr, const int32_t* s_indices,
                       const double* s_values, int64_t m, const int64_t* p_indptr, const int32_t* p_indices,
                       const float* p_values, const int64_t* seen_indptr, const int32_t* seen_indices, int implicit,
                       int k, int acc_rows, int64_t* out_nnz, int64_t* out_dense, int64_t* out_sparse,
                       double* out_scores);

/* res[i0,:,:] += val * U[i1,:] (x) W[i2,:] over all nnz of a 3-way COO tensor sorted
 * and grouped by mode-0 index (CSR-like: seg_ptr int64 [n0+1], i1/i2 int32 [nnz]);
 * out [n0 x ru*rw] row-major (ld = ldo).  Replaces dttm_seq/dttm_par,
 * polara/lib/sparse.py:203-234. */
int pb200_ttm(pb200_ctx* ctx, int64_t n0, int64_t nnz, const int64_t* seg_ptr,
              const int32_t* i1, const int32_t* i2, const float* values,
              const float* U, int ru, int64_t ldu, const float* W, int rw, int64_t ldw,
              float* out, int64_t ldo);

/* Same sum when the grouped mode has only a few huge segments (the feedback mode of the
 * user x item x feedback tensor): out[s, x*rb + y] = sum_{p in segment s} val_p A[ia_p,x] B[ib_p,y],
 * fp64 accumulation, deterministic.  seg_ptr int64 [n_seg+1] (device).  Synchronises the stream. */
int pb200_ttm_reduce(pb200_ctx* ctx, int n_seg, int64_t nnz, const int64_t* seg_ptr,
                     const int32_t* ia, const int32_t* ib, const float* values,
                     const float* A, int ra, int64_t lda, const float* B, int rb, int64_t ldb,
                     float* out, int64_t ldo);

/* Stable grouping of a 3-way COO tensor by one mode: nnz sorted by key (0..n_keys-1);
 * seg_ptr int64 [n_keys+1]; a_out/b_out/val_out = the other index arrays / values permuted.
 * arrange_indices (polara/lib/sparse.py:239-264) is the reference's host-side analogue. */
int pb200_coo_group(pb200_ctx* ctx, int64_t nnz, int64_t n_keys, const int32_t* key,
                    const int32_t* a, const int32_t* b, const float* val,
                    int64_t* seg_ptr, int32_t* a_out, int32_t* b_out, float* val_out);

/* out[n x ldo] (float32) = fp32(V R) for V fp64 [n x K] (ldv) and R fp64 [K x r] (ldr), 1 <= K, r <= 1024; columns
 * r..ldo-1 are zero.  Each element is acc = 0.0, acc = __dadd_rn(acc, __dmul_rn(V[i,k], R[k,j])) for k ascending, then
 * __double2float_rn(acc).  The factor rotation of CoffeeModel._check_reduced_rank (models.py:949-963:
 * factor.dot(rotation)) for the item factor of the Tucker-rank sweep. */
int pb200_rotate_factor(pb200_ctx* ctx, int64_t n, int K, int r, const double* V, int64_t ldv,
                        const double* R, int64_t ldr, float* out, int64_t ldo);

#ifdef __cplusplus
}
#endif
#endif

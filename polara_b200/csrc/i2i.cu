// Item-to-item (co-occurrence) model, CooccurrenceModel of polara/recommender/models.py:693-725:
//   pb200_cooc_build  S = A^T A in fp64 with a zero diagonal (models.py:702-709), dense [n x lds];
//   pb200_i2i_topk    per test user s_u = sum_i p_ui S[i, :] (lib/sparse.py:35-55 as scipy's csr_matmat sums it), its
//                     nonzero count and its top-k lists under the dense and the sparse chunk rule (models.py:494-563).
// Summation orders are fixed (no atomics), so every result is deterministic; see DESIGN.md section 3.5.
#include "common.cuh"

#include <algorithm>

#include <cub/device/device_radix_sort.cuh>
#include <math_constants.h>

namespace {

constexpr int kBuildThreads = 128;       // threads of one build CTA (one item row, one column panel)
constexpr int kBuildBatch = 128;         // users whose slice bounds one CTA stages in shared memory at a time
constexpr int kScoreR = 8;               // fp64 accumulators per lane: one warp holds a panel of 32 * kScoreR columns

__device__ __forceinline__ float sgn(float x) { return (float)((x > 0.f) - (x < 0.f)); }

// ---- build ----------------------------------------------------------------------------------------------------------
// work of item row i: sum over its users of their row lengths (the number of products the row's CTAs make)
__global__ void row_work_kernel(const int64_t* __restrict__ at_indptr, const int32_t* __restrict__ at_indices,
                                const int64_t* __restrict__ a_indptr, int64_t n, uint64_t* __restrict__ work,
                                int32_t* __restrict__ iota) {
    const int lane = threadIdx.x & 31;
    const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n) return;
    uint64_t w = 0;
    for (int64_t q = at_indptr[i] + lane; q < at_indptr[i + 1]; q += 32) {
        const int u = at_indices[q];
        w += (uint64_t)(a_indptr[u + 1] - a_indptr[u]);
    }
    for (int o = 16; o > 0; o >>= 1) w += __shfl_xor_sync(0xffffffffu, w, o);
    if (lane == 0) { work[i] = w; iota[i] = (int32_t)i; }
}

// One CTA per (item row i, column panel p).  The row panel S[i, c0 : c0 + w) lives in shared memory; the users of
// column i of A are taken in ascending order and each adds a_ui * a_uj for the items j of its row in the panel.  A
// user's items are distinct, so within one user no two threads touch the same entry; a barrier separates the users,
// so every entry is summed over the users in ascending order.  fp32 * fp32 is exact in fp64.
// A is panel-major (pb200_csr_block_columns): virtual row p * m + u holds the items of row u inside panel p.
__global__ void __launch_bounds__(kBuildThreads)
cooc_build_kernel(int64_t n, int64_t m, int64_t panel_cols, int n_panels, const int64_t* __restrict__ a_indptr,
                  const int32_t* __restrict__ a_indices, const float* __restrict__ a_values,
                  const int64_t* __restrict__ at_indptr, const int32_t* __restrict__ at_indices,
                  const float* __restrict__ at_values, const int32_t* __restrict__ row_order, int implicit,
                  double* __restrict__ S, int64_t lds) {
    extern __shared__ double acc[];
    __shared__ int64_t s_beg[kBuildBatch], s_end[kBuildBatch];
    __shared__ float s_x[kBuildBatch];
    const int64_t i = row_order[blockIdx.x / n_panels];
    const int p = blockIdx.x % n_panels;
    const int64_t c0 = (int64_t)p * panel_cols;
    const int w = (int)min(panel_cols, n - c0);
    for (int t = threadIdx.x; t < w; t += blockDim.x) acc[t] = 0.0;
    const int64_t qb = at_indptr[i], qe = at_indptr[i + 1];
    for (int64_t q0 = qb; q0 < qe; q0 += kBuildBatch) {
        const int nb = (int)min((int64_t)kBuildBatch, qe - q0);
        __syncthreads();                 // the previous batch's bounds are consumed (first pass: acc is cleared)
        for (int t = threadIdx.x; t < nb; t += blockDim.x) {
            const int64_t u = at_indices[q0 + t];
            const float x = at_values[q0 + t];
            s_beg[t] = a_indptr[p * m + u];
            s_end[t] = a_indptr[p * m + u + 1];
            s_x[t] = implicit ? sgn(x) : x;
        }
        __syncthreads();
        for (int b = 0; b < nb; ++b) {
            const int64_t e = s_end[b];
            if (s_beg[b] == e) continue;                    // uniform: no barrier needed for an empty slice
            const double x = (double)s_x[b];
            for (int64_t t = s_beg[b] + threadIdx.x; t < e; t += blockDim.x) {
                const float y = a_values[t];
                const int j = (int)(a_indices[t] - c0);
                acc[j] = __dadd_rn(acc[j], __dmul_rn(x, (double)(implicit ? sgn(y) : y)));
            }
            __syncthreads();
        }
    }
    __syncthreads();
    double* row = S + i * lds + c0;
    for (int t = threadIdx.x; t < w; t += blockDim.x) row[t] = (c0 + t == i) ? 0.0 : acc[t];    // setdiag(0), :706
}

// ---- scoring ----------------------------------------------------------------------------------------------------------
struct ICand { double score; int32_t id; int32_t seen; };

// (seen asc, score desc, id asc): the dense rule with seen items after all unseen ones; seen is 0 for the sparse rule
__device__ __forceinline__ bool ibefore(double sa, int ia, int fa, double sb, int ib, int fb) {
    return fa < fb || (fa == fb && (sa > sb || (sa == sb && ia < ib)));
}

// warp-cooperative insertion into a sorted list of capacity cap and fill cnt (warp-uniform); returns the new fill
__device__ __forceinline__ int ilist_insert(ICand* list, int cap, int cnt, double s, int id, int f, int lane) {
    if (cnt == cap) {
        const ICand last = list[cap - 1];
        if (!ibefore(s, id, f, last.score, last.id, last.seen)) return cnt;
    }
    int pos = 0;
    for (int base = 0; base < cnt; base += 32) {
        const int i = base + lane;
        bool b = false;
        if (i < cnt) { const ICand c = list[i]; b = ibefore(c.score, c.id, c.seen, s, id, f); }
        pos += __popc(__ballot_sync(0xffffffffu, b));
    }
    for (int hi = min(cnt, cap - 1); hi > pos; hi -= 32) {
        const int dst = hi - lane;
        ICand c;
        const bool act = dst > pos;
        if (act) c = list[dst - 1];
        __syncwarp();
        if (act) list[dst] = c;
        __syncwarp();
    }
    if (lane == 0) { ICand c; c.score = s; c.id = id; c.seen = f; list[pos] = c; }
    __syncwarp();
    return min(cnt + 1, cap);
}

__device__ __forceinline__ bool in_sorted(const int32_t* __restrict__ a, int64_t beg, int64_t end, int key) {
    int64_t lo = beg, hi = end;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(a + mid) < key) lo = mid + 1; else hi = mid;
    }
    return lo < end && __ldg(a + lo) == key;
}

__global__ void row_len_kernel(const int64_t* __restrict__ indptr, int64_t m, uint32_t* __restrict__ len,
                               int32_t* __restrict__ iota) {
    const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= m) return;
    len[u] = (uint32_t)min(indptr[u + 1] - indptr[u], (int64_t)0xffffffffll);
    iota[u] = (int32_t)u;
}

// One warp per test user (users handed out longest row first).  The warp sweeps the item axis in panels of
// 32 * kScoreR columns; lane l owns columns c0 + r * 32 + l.  Per panel the user's items i are taken in ascending order
// and acc = dadd(acc, dmul(p_ui, S[i, col])) -- a rounded product, then a rounded sum, as csr_matmat forms it -- so each
// S row of the user is read once in all.  The finished panel is offered to both lists in ascending column order.
__global__ void __launch_bounds__(256)
i2i_topk_kernel(const double* __restrict__ S, int64_t lds, int64_t n, int64_t m, const int64_t* __restrict__ p_indptr,
                const int32_t* __restrict__ p_indices, const float* __restrict__ p_values,
                const int64_t* __restrict__ seen_indptr, const int32_t* __restrict__ seen_indices, int implicit, int k,
                const int32_t* __restrict__ user_order, ICand* __restrict__ lists, int64_t* __restrict__ out_nnz,
                int64_t* __restrict__ out_dense, int64_t* __restrict__ out_sparse, double* __restrict__ out_scores) {
    __shared__ double s_panel[8][32 * kScoreR];
    const int lane = threadIdx.x & 31;
    const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= m) return;
    double* panel = s_panel[threadIdx.x >> 5];
    const int64_t u = user_order[w];
    ICand* dl = lists + u * 2 * k;        // dense rule
    ICand* sl = dl + k;                   // sparse rule
    const int64_t pb = p_indptr[u], pe = p_indptr[u + 1];
    int64_t sb = 0, se = 0;
    if (seen_indptr) { sb = seen_indptr[u]; se = seen_indptr[u + 1]; }
    int cd = 0, cs = 0;                   // fills
    double td = 0.0, ts = 0.0;            // last entries' scores once full
    int fd = 0;                           // last dense entry is a seen item
    int64_t nnz = 0;
    for (int64_t c0 = 0; c0 < n; c0 += 32 * kScoreR) {
        double acc[kScoreR];
#pragma unroll
        for (int r = 0; r < kScoreR; ++r) acc[r] = 0.0;
        for (int64_t q0 = pb; q0 < pe; q0 += 32) {
            int my_i = 0;
            float my_p = 0.f;
            if (q0 + lane < pe) { my_i = p_indices[q0 + lane]; my_p = p_values[q0 + lane]; }
            if (implicit) my_p = sgn(my_p);
            const int nq = (int)min((int64_t)32, pe - q0);
            for (int t = 0; t < nq; ++t) {
                const int i = __shfl_sync(0xffffffffu, my_i, t);
                const double pv = (double)__shfl_sync(0xffffffffu, my_p, t);
                const double* row = S + (int64_t)i * lds + c0 + lane;
                double v[kScoreR];
#pragma unroll
                for (int r = 0; r < kScoreR; ++r) v[r] = (c0 + r * 32 + lane < n) ? __ldg(row + r * 32) : 0.0;
#pragma unroll
                for (int r = 0; r < kScoreR; ++r) acc[r] = __dadd_rn(acc[r], __dmul_rn(pv, v[r]));
            }
        }
        // the candidate pass runs from shared memory so that its insertion code is not unrolled kScoreR times
#pragma unroll
        for (int r = 0; r < kScoreR; ++r) panel[r * 32 + lane] = acc[r];
        __syncwarp();
#pragma unroll 1
        for (int r = 0; r < kScoreR; ++r) {
            const int64_t base = c0 + r * 32;
            if (base >= n) break;
            const int64_t j = base + lane;
            const bool valid = j < n;
            const double x = panel[r * 32 + lane];
            nnz += (valid && x != 0.0);
            // cheap screens first; the seen lookup only for what survives them
            const bool maybe_d = valid && (cd < k || fd || x > td);
            const bool maybe_s = valid && x != 0.0 && (cs < k || x > ts);
            int seen = 0;
            if (maybe_d && sb < se) seen = in_sorted(seen_indices, sb, se, (int)j);
            // ids ascend along the sweep: an equal score later never displaces an earlier entry of the same flag
            const bool pass_d = maybe_d && (cd < k || (fd ? (!seen || x > td) : (!seen && x > td)));
            const bool pass_s = maybe_s;       // the reference's sparse blocks keep the seen scores (see the header)
            unsigned mask = __ballot_sync(0xffffffffu, pass_d);
            while (mask) {
                const int t = __ffs(mask) - 1;
                mask &= mask - 1;
                cd = ilist_insert(dl, k, cd, __shfl_sync(0xffffffffu, x, t), (int)(base + t),
                                  __shfl_sync(0xffffffffu, seen, t), lane);
                if (cd == k) { const ICand last = dl[k - 1]; td = last.score; fd = last.seen; }
            }
            mask = __ballot_sync(0xffffffffu, pass_s);
            while (mask) {
                const int t = __ffs(mask) - 1;
                mask &= mask - 1;
                cs = ilist_insert(sl, k, cs, __shfl_sync(0xffffffffu, x, t), (int)(base + t), 0, lane);
                if (cs == k) ts = sl[k - 1].score;
            }
        }
    }
    for (int o = 16; o > 0; o >>= 1) nnz += __shfl_xor_sync(0xffffffffu, nnz, o);
    if (lane == 0) out_nnz[u] = nnz;
    for (int i = lane; i < k; i += 32) {
        out_dense[u * k + i] = i < cd ? (int64_t)dl[i].id : -1;
        if (out_scores) out_scores[u * k + i] = i < cd ? dl[i].score : -CUDART_INF;
        out_sparse[u * k + i] = i < cs ? (int64_t)sl[i].id : -1;        // _pad_const, models.py:73, 531-533
    }
}

// descending sort of `key` carrying `iota` (the launch order of the rows / users)
template <typename K>
int sort_desc(pb200_ctx* ctx, Scratch& sc, const K* key, const int32_t* iota, int64_t count, int32_t* order) {
    K* key_sorted = nullptr;
    void* temp = nullptr;
    size_t temp_bytes = 0;
    PB_TRY(sc.alloc(&key_sorted, (size_t)count));
    PB_CUDA(ctx, cub::DeviceRadixSort::SortPairsDescending(nullptr, temp_bytes, key, key_sorted, iota, order, count, 0,
                                                           (int)(8 * sizeof(K)), ctx->stream));
    PB_TRY(sc.alloc(reinterpret_cast<char**>(&temp), temp_bytes));
    PB_CUDA(ctx, cub::DeviceRadixSort::SortPairsDescending(temp, temp_bytes, key, key_sorted, iota, order, count, 0,
                                                           (int)(8 * sizeof(K)), ctx->stream));
    return PB200_OK;
}

}  // namespace

extern "C" int pb200_cooc_build(pb200_ctx* ctx, const pb200_csr_view* a, const pb200_csr_view* at, int implicit,
                                double* S, int64_t lds) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, a != nullptr && at != nullptr && S != nullptr, "cooc_build: null argument");
    const int64_t m = a->n_rows, n = a->n_cols;
    PB_REQUIRE(ctx, n > 0 && m >= 0 && n < (int64_t)2147483647 && m < (int64_t)2147483647, "cooc_build: bad shape");
    PB_REQUIRE(ctx, at->n_rows == n && at->n_cols == m && at->nnz == a->nnz && at->n_panels == 1,
               "cooc_build: `at` must be the plain CSR of A^T (pb200_csr_transpose)");
    PB_REQUIRE(ctx, lds >= n, "cooc_build: lds < n_items");
    PB_REQUIRE(ctx, a->n_panels >= 1 && a->panel_cols * (int64_t)sizeof(double) <= PB200_COOC_MAX_PANEL_BYTES &&
                        (int64_t)a->n_panels == std::max<int64_t>(1, ceil_div64(n, a->panel_cols)),
               "cooc_build: A must be split into column panels of at most PB200_COOC_MAX_PANEL_BYTES / 8 columns "
               "(pb200_csr_block_columns)");
    PB_REQUIRE(ctx, n * (int64_t)a->n_panels < (int64_t)2147483647, "cooc_build: too many (row, panel) blocks");
    Scratch sc(ctx);
    uint64_t* work = nullptr;
    int32_t *iota = nullptr, *order = nullptr;
    PB_TRY(sc.alloc(&work, (size_t)n));
    PB_TRY(sc.alloc(&iota, (size_t)n));
    PB_TRY(sc.alloc(&order, (size_t)n));
    row_work_kernel<<<(unsigned)ceil_div64(n * 32, 256), 256, 0, ctx->stream>>>(at->indptr, at->indices, a->indptr, n,
                                                                               work, iota);
    PB_TRY(sort_desc(ctx, sc, work, iota, n, order));                // longest rows first
    const size_t smem = (size_t)std::min<int64_t>(a->panel_cols, n) * sizeof(double);
    PB_CUDA(ctx, cudaFuncSetAttribute(cooc_build_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cooc_build_kernel<<<(unsigned)(n * a->n_panels), kBuildThreads, smem, ctx->stream>>>(
        n, m, a->panel_cols, a->n_panels, a->indptr, a->indices, a->values, at->indptr, at->indices, at->values, order,
        implicit ? 1 : 0, S, lds);
    ctx->stats[0] += 2;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

extern "C" int pb200_i2i_topk(pb200_ctx* ctx, const double* S, int64_t lds, int64_t n, int64_t m,
                              const int64_t* p_indptr, const int32_t* p_indices, const float* p_values,
                              const int64_t* seen_indptr, const int32_t* seen_indices, int implicit, int k,
                              int64_t* out_nnz, int64_t* out_dense, int64_t* out_sparse, double* out_scores) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, n > 0 && m >= 0 && lds >= n && n < (int64_t)2147483647, "i2i_topk: bad shape");
    PB_REQUIRE(ctx, k > 0 && k <= n, "i2i_topk: k must be in 1..n_items");
    PB_REQUIRE(ctx, S != nullptr && p_indptr != nullptr && out_nnz != nullptr && out_dense != nullptr &&
                        out_sparse != nullptr, "i2i_topk: null argument");
    PB_REQUIRE(ctx, (seen_indptr == nullptr) == (seen_indices == nullptr), "i2i_topk: seen CSR must be both or neither");
    if (m == 0) return PB200_OK;
    PB_REQUIRE(ctx, m < (int64_t)2147483647, "i2i_topk: too many users");
    Scratch sc(ctx);
    uint32_t* len = nullptr;
    int32_t *iota = nullptr, *order = nullptr;
    ICand* lists = nullptr;
    PB_TRY(sc.alloc(&len, (size_t)m));
    PB_TRY(sc.alloc(&iota, (size_t)m));
    PB_TRY(sc.alloc(&order, (size_t)m));
    PB_TRY(sc.alloc(&lists, (size_t)m * 2 * k));
    row_len_kernel<<<(unsigned)ceil_div64(m, 256), 256, 0, ctx->stream>>>(p_indptr, m, len, iota);
    PB_TRY(sort_desc(ctx, sc, len, iota, m, order));                  // longest test rows first
    i2i_topk_kernel<<<(unsigned)ceil_div64(m * 32, 256), 256, 0, ctx->stream>>>(
        S, lds, n, m, p_indptr, p_indices, p_values, seen_indptr, seen_indices, implicit ? 1 : 0, k, order, lists,
        out_nnz, out_dense, out_sparse, out_scores);
    ctx->stats[0] += 2;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

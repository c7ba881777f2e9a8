// Item-to-item (co-occurrence) model, CooccurrenceModel of polara/recommender/models.py:693-725:
//   pb200_cooc_build  S = A^T A in fp64 with a zero diagonal (models.py:702-709), dense [n x lds];
//   pb200_i2i_topk    per test user s_u = sum_i p_ui S[i, :] (lib/sparse.py:35-55 as scipy's csr_matmat sums it), its
//                     nonzero count and its top-k lists under the dense and the sparse chunk rule (models.py:494-563).
//   pb200_cooc_build_csr  the same S as an fp64 CSR (two passes: exact row counts, then the rows), for catalogues whose
//                         dense S does not fit;
//   pb200_i2i_topk_csr    pb200_i2i_topk on a CSR S, bit-equal to it on the same S.
// Summation orders are fixed (no atomics), so every result is deterministic; see DESIGN.md section 3.5.
#include "common.cuh"

#include <algorithm>

#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
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

// ---- sparse S ---------------------------------------------------------------------------------------------------------
// A row of S (build) or of P S (scoring) is accumulated in one of two places, chosen by its work w (the number of products
// that form it, an upper bound on its distinct columns):
//   w <= kHashWork  a per-warp open-addressing table in shared memory of cap = pow2 >= 2w slots (load <= 1/2);
//   otherwise       a dense fp64 row of n entries in global scratch, one per CTA (build) or warp (scoring), zero between
//                   uses.
// Either way an entry is summed in the order of the dense kernels, so it has their bits.
constexpr int kHashSlots = 1024;          // slots of one warp's table: 1024 * (4 + 8) B = 12 KB
constexpr int kHashWork = kHashSlots / 2;
constexpr int kSparseWarps = 8;           // warps per CTA of the table kernels: 96 KB of dynamic shared memory
constexpr int kLongThreads = 256;         // threads of one build CTA on the global-row path
constexpr int kEmpty = 0x7fffffff;        // empty slot; sorts after every column id

__device__ __forceinline__ int table_cap(uint64_t w) {
    int cap = 32;
    while ((uint64_t)cap < 2 * w) cap <<= 1;
    return cap;
}

__device__ __forceinline__ int slot_hash(int j, int cap) { return (int)(((uint32_t)j * 2654435761u) & (uint32_t)(cap - 1)); }

// the slot of column j, claimed if j is new; distinct lanes insert distinct columns, so a claimed slot is never shared
__device__ __forceinline__ int table_insert(int* keys, int cap, int j) {
    int h = slot_hash(j, cap);
    while (true) {
        const int k = keys[h];
        if (k == j) return h;
        if (k == kEmpty) {
            const int old = atomicCAS(keys + h, kEmpty, j);
            if (old == kEmpty || old == j) return h;
        }
        h = (h + 1) & (cap - 1);
    }
}

__device__ __forceinline__ double table_get(const int* keys, const double* vals, int cap, int j) {
    int h = slot_hash(j, cap);
    while (true) {
        const int k = keys[h];
        if (k == j) return vals[h];
        if (k == kEmpty) return 0.0;
        h = (h + 1) & (cap - 1);
    }
}

__device__ __forceinline__ void table_clear(int* keys, double* vals, int cap, int lane) {
    for (int t = lane; t < cap; t += 32) { keys[t] = kEmpty; vals[t] = 0.0; }
    __syncwarp();
}

// warp-wide bitonic sort of the table by key (cap is a power of two): the occupied slots come first, ascending
__device__ void table_sort(int* keys, double* vals, int cap, int lane) {
    for (int size = 2; size <= cap; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = lane; t < cap / 2; t += 32) {
                const int lo = 2 * t - (t & (stride - 1));
                const int hi = lo + stride;
                const bool asc = (lo & size) == 0;
                const int ka = keys[lo], kb = keys[hi];
                if ((ka > kb) == asc) {
                    keys[lo] = kb; keys[hi] = ka;
                    const double v = vals[lo]; vals[lo] = vals[hi]; vals[hi] = v;
                }
            }
            __syncwarp();
        }
    }
}

// Build, table path: one warp per item row i with work <= kHashWork (rows in the longest-first order; longer rows are
// left to cooc_csr_long_kernel).  The users of column i are taken in ascending order and a barrier separates them, as in
// cooc_build_kernel.  kFill = false: count[i] = the row's entries that are not exactly 0; kFill = true: the row, sorted
// by column, at indptr[i].
template <bool kFill>
__global__ void __launch_bounds__(32 * kSparseWarps)
cooc_csr_table_kernel(int64_t n, const int64_t* __restrict__ a_indptr, const int32_t* __restrict__ a_indices,
                      const float* __restrict__ a_values, const int64_t* __restrict__ at_indptr,
                      const int32_t* __restrict__ at_indices, const float* __restrict__ at_values,
                      const int32_t* __restrict__ row_order, const uint64_t* __restrict__ work, int implicit,
                      int64_t* __restrict__ count, const int64_t* __restrict__ indptr, int32_t* __restrict__ out_idx,
                      double* __restrict__ out_val) {
    extern __shared__ double smem_d[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    double* vals = smem_d + wib * kHashSlots;
    int* keys = reinterpret_cast<int*>(smem_d + kSparseWarps * kHashSlots) + wib * kHashSlots;
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= n) return;
    const int i = row_order[r];
    const uint64_t w = work[i];
    if (w > (uint64_t)kHashWork) return;
    const int cap = table_cap(w);
    table_clear(keys, vals, cap, lane);
    const int64_t qb = at_indptr[i], qe = at_indptr[i + 1];
    for (int64_t q0 = qb; q0 < qe; q0 += 32) {
        int my_u = 0;
        float my_x = 0.f;
        if (q0 + lane < qe) { my_u = at_indices[q0 + lane]; my_x = at_values[q0 + lane]; }
        const int nq = (int)min((int64_t)32, qe - q0);
        for (int t = 0; t < nq; ++t) {
            const int u = __shfl_sync(0xffffffffu, my_u, t);
            const float xf = __shfl_sync(0xffffffffu, my_x, t);
            const double x = (double)(implicit ? sgn(xf) : xf);
            const int64_t e1 = a_indptr[u + 1];
            for (int64_t e = a_indptr[u] + lane; e < e1; e += 32) {
                const int j = a_indices[e];
                if (j == i) continue;                                   // setdiag(0)
                const float y = a_values[e];
                const int s = table_insert(keys, cap, j);
                vals[s] = __dadd_rn(vals[s], __dmul_rn(x, (double)(implicit ? sgn(y) : y)));
            }
            __syncwarp();
        }
    }
    if (!kFill) {
        int c = 0;
        for (int t = lane; t < cap; t += 32) c += (keys[t] != kEmpty && vals[t] != 0.0);
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) count[i] = c;
        return;
    }
    table_sort(keys, vals, cap, lane);
    int64_t dst = indptr[i];
    for (int t0 = 0; t0 < cap; t0 += 32) {
        const int t = t0 + lane;
        const int key = keys[t];
        const double v = vals[t];
        const bool keep = key != kEmpty && v != 0.0;                    // eliminate_zeros()
        const unsigned mask = __ballot_sync(0xffffffffu, keep);
        if (keep) {
            const int64_t at = dst + __popc(mask & ((1u << lane) - 1u));
            out_idx[at] = key;
            out_val[at] = v;
        }
        dst += __popc(mask);
        if (keys[t0 + 31] == kEmpty) break;                             // sorted: nothing occupied after this
    }
}

// Build, global-row path: each CTA takes the rows with work > kHashWork at positions blockIdx.x, + gridDim.x, ... of the
// longest-first order and accumulates them in its own zeroed row acc[0, n) exactly as cooc_build_kernel does its panel.
// The row is then read in column order -- the output comes out sorted -- and cleared behind the read.
template <bool kFill>
__global__ void __launch_bounds__(kLongThreads)
cooc_csr_long_kernel(int64_t n, const int64_t* __restrict__ a_indptr, const int32_t* __restrict__ a_indices,
                     const float* __restrict__ a_values, const int64_t* __restrict__ at_indptr,
                     const int32_t* __restrict__ at_indices, const float* __restrict__ at_values,
                     const int32_t* __restrict__ row_order, const uint64_t* __restrict__ work, int implicit,
                     double* __restrict__ acc_rows, int64_t* __restrict__ count, const int64_t* __restrict__ indptr,
                     int32_t* __restrict__ out_idx, double* __restrict__ out_val) {
    using Scan = cub::BlockScan<int, kLongThreads>;
    __shared__ typename Scan::TempStorage scan_tmp;
    __shared__ int64_t s_beg[kBuildBatch], s_end[kBuildBatch];
    __shared__ float s_x[kBuildBatch];
    double* acc = acc_rows + (int64_t)blockIdx.x * n;
    for (int64_t r = blockIdx.x; r < n; r += gridDim.x) {
        const int i = row_order[r];
        if (work[i] <= (uint64_t)kHashWork) break;                      // the rest are table rows
        const int64_t qb = at_indptr[i], qe = at_indptr[i + 1];
        for (int64_t q0 = qb; q0 < qe; q0 += kBuildBatch) {
            const int nb = (int)min((int64_t)kBuildBatch, qe - q0);
            __syncthreads();
            for (int t = threadIdx.x; t < nb; t += blockDim.x) {
                const int64_t u = at_indices[q0 + t];
                const float x = at_values[q0 + t];
                s_beg[t] = a_indptr[u];
                s_end[t] = a_indptr[u + 1];
                s_x[t] = implicit ? sgn(x) : x;
            }
            __syncthreads();
            for (int b = 0; b < nb; ++b) {
                const int64_t e = s_end[b];
                if (s_beg[b] == e) continue;
                const double x = (double)s_x[b];
                for (int64_t t = s_beg[b] + threadIdx.x; t < e; t += blockDim.x) {
                    const int j = a_indices[t];
                    if (j == i) continue;
                    const float y = a_values[t];
                    acc[j] = __dadd_rn(acc[j], __dmul_rn(x, (double)(implicit ? sgn(y) : y)));
                }
                __syncthreads();
            }
        }
        __syncthreads();
        int64_t dst = kFill ? indptr[i] : 0;
        int64_t total = 0;
        for (int64_t c0 = 0; c0 < n; c0 += kLongThreads) {
            const int64_t j = c0 + threadIdx.x;
            double v = 0.0;
            if (j < n) {
                v = acc[j];
                if (v != 0.0) acc[j] = 0.0;
            }
            const int keep = v != 0.0;
            int off, agg;
            Scan(scan_tmp).ExclusiveSum(keep, off, agg);
            if (kFill && keep) { out_idx[dst + off] = (int32_t)j; out_val[dst + off] = v; }
            dst += agg;
            total += agg;
            __syncthreads();                                            // scan_tmp is reused
        }
        if (!kFill && threadIdx.x == 0) count[i] = total;
    }
}

// number of entries with work > kHashWork (the rows / users of the global-row path)
__global__ void count_long_kernel(const uint64_t* __restrict__ work, int64_t count, unsigned long long* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned mask = __ballot_sync(0xffffffffu, i < count && work[i] > (uint64_t)kHashWork);
    if ((threadIdx.x & 31) == 0 && mask) atomicAdd(out, (unsigned long long)__popc(mask));
}

// the count of count_long_kernel, on the host (one readback: it sizes the global rows before they are allocated)
int count_long(pb200_ctx* ctx, Scratch& sc, const uint64_t* work, int64_t count, int64_t* host_out) {
    unsigned long long* d = nullptr;
    PB_TRY(sc.alloc(&d, 1));
    PB_CUDA(ctx, cudaMemsetAsync(d, 0, sizeof(unsigned long long), ctx->stream));
    count_long_kernel<<<(unsigned)ceil_div64(count, 256), 256, 0, ctx->stream>>>(work, count, d);
    unsigned long long h = 0;
    PB_CUDA(ctx, cudaMemcpyAsync(&h, d, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
    PB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *host_out = (int64_t)h;
    return PB200_OK;
}

// ---- scoring on a sparse S ---------------------------------------------------------------------------------------------
struct ListState {
    int cd = 0, cs = 0;                   // fills of the dense-rule and the sparse-rule list
    double td = 0.0, ts = 0.0;            // their last entries once full
    int id_d = 0, id_s = 0, fd = 0;
};

// Offers one nonzero score per lane (valid) to both lists.  The touched entries come in no particular column order, so
// the screens compare the full (seen, score desc, id asc) key.
__device__ __forceinline__ void offer_scores(ICand* dl, ICand* sl, int k, ListState& st, double x, int j, bool valid,
                                             const int32_t* __restrict__ seen_indices, int64_t sb, int64_t se,
                                             int lane) {
    const bool maybe_d = valid && (st.cd < k || st.fd || x > st.td || (x == st.td && j < st.id_d));
    const bool maybe_s = valid && (st.cs < k || x > st.ts || (x == st.ts && j < st.id_s));
    int seen = 0;
    if (maybe_d && sb < se) seen = in_sorted(seen_indices, sb, se, j);
    const bool pass_d = maybe_d && (st.cd < k || ibefore(x, j, seen, st.td, st.id_d, st.fd));
    unsigned mask = __ballot_sync(0xffffffffu, pass_d);
    while (mask) {
        const int t = __ffs(mask) - 1;
        mask &= mask - 1;
        st.cd = ilist_insert(dl, k, st.cd, __shfl_sync(0xffffffffu, x, t), __shfl_sync(0xffffffffu, j, t),
                             __shfl_sync(0xffffffffu, seen, t), lane);
        if (st.cd == k) { const ICand last = dl[k - 1]; st.td = last.score; st.id_d = last.id; st.fd = last.seen; }
    }
    mask = __ballot_sync(0xffffffffu, maybe_s);
    while (mask) {
        const int t = __ffs(mask) - 1;
        mask &= mask - 1;
        st.cs = ilist_insert(sl, k, st.cs, __shfl_sync(0xffffffffu, x, t), __shfl_sync(0xffffffffu, j, t), 0, lane);
        if (st.cs == k) { const ICand last = sl[k - 1]; st.ts = last.score; st.id_s = last.id; }
    }
}

// The dense rule from the list of nonzero scores: within each class (unseen, then seen; one class without a seen CSR) the
// positive scores, then the items whose score is exactly 0 by ascending id, then the negative scores -- the order of
// (seen, score desc, id asc) over all n items.  score(j) returns the user's score of item j.
template <class Score>
__device__ void write_dense_list(const Score& score, const ICand* dl, int cd, int k, int64_t n,
                                 const int32_t* __restrict__ seen_indices, int64_t sb, int64_t se, bool has_seen,
                                 int64_t* __restrict__ out, double* __restrict__ out_sc, int lane) {
    int pos = 0, idx = 0;
    for (int f = 0; f < (has_seen ? 2 : 1) && pos < k; ++f) {
        for (; pos < k && idx < cd && dl[idx].seen == f && dl[idx].score > 0.0; ++pos, ++idx) {
            if (lane == 0) { out[pos] = dl[idx].id; if (out_sc) out_sc[pos] = dl[idx].score; }
        }
        // zero scores of class f by ascending id: unseen ones from the whole catalogue, seen ones from the seen row
        const int64_t lim = f == 0 ? n : se - sb;
        for (int64_t c0 = 0; c0 < lim && pos < k; c0 += 32) {
            const int64_t c = c0 + lane;
            bool z = false;
            int j = 0;
            if (c < lim) {
                j = f == 0 ? (int)c : __ldg(seen_indices + sb + c);
                z = score(j) == 0.0 && (f == 1 || !has_seen || !in_sorted(seen_indices, sb, se, j));
            }
            const unsigned mask = __ballot_sync(0xffffffffu, z);
            const int at = pos + __popc(mask & ((1u << lane) - 1u));
            if (z && at < k) { out[at] = j; if (out_sc) out_sc[at] = 0.0; }
            pos = min(k, pos + __popc(mask));
        }
        for (; pos < k && idx < cd && dl[idx].seen == f; ++pos, ++idx) {
            if (lane == 0) { out[pos] = dl[idx].id; if (out_sc) out_sc[pos] = dl[idx].score; }
        }
    }
    __syncwarp();
}

struct TableScore {
    const int* keys; const double* vals; int cap;
    __device__ double operator()(int j) const { return table_get(keys, vals, cap, j); }
};
struct RowScore {
    const double* row;
    __device__ double operator()(int j) const { return row[j]; }
};

__device__ __forceinline__ void write_outputs(const ICand* sl, int cs, int64_t nnz, int k, int64_t u,
                                              int64_t* __restrict__ out_nnz, int64_t* __restrict__ out_sparse, int lane) {
    for (int o = 16; o > 0; o >>= 1) nnz += __shfl_xor_sync(0xffffffffu, nnz, o);
    if (lane == 0) out_nnz[u] = nnz;
    for (int i = lane; i < k; i += 32) out_sparse[u * k + i] = i < cs ? (int64_t)sl[i].id : -1;
}

// Scoring, table path: one warp per test user with work (sum of nnz of its S rows) <= kHashWork.  The user's items i are
// taken in ascending order and acc[j] = dadd(acc[j], dmul(p_ui, S[i, j])) over row i of S, a warp barrier between the
// rows: the dense kernel's sequence with its zero terms left out (adding +-0 to a sum changes none of its bits).
__global__ void __launch_bounds__(32 * kSparseWarps)
i2i_csr_table_kernel(int64_t n, int64_t m, const int64_t* __restrict__ s_indptr, const int32_t* __restrict__ s_indices,
                     const double* __restrict__ s_values, const int64_t* __restrict__ p_indptr,
                     const int32_t* __restrict__ p_indices, const float* __restrict__ p_values,
                     const int64_t* __restrict__ seen_indptr, const int32_t* __restrict__ seen_indices, int implicit,
                     int k, const int32_t* __restrict__ user_order, const uint64_t* __restrict__ work,
                     ICand* __restrict__ lists, int64_t* __restrict__ out_nnz, int64_t* __restrict__ out_dense,
                     int64_t* __restrict__ out_sparse, double* __restrict__ out_scores) {
    extern __shared__ double smem_d[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    double* vals = smem_d + wib * kHashSlots;
    int* keys = reinterpret_cast<int*>(smem_d + kSparseWarps * kHashSlots) + wib * kHashSlots;
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= m) return;
    const int64_t u = user_order[r];
    const uint64_t w = work[u];
    if (w > (uint64_t)kHashWork) return;
    const int cap = table_cap(w);
    table_clear(keys, vals, cap, lane);
    const int64_t pb = p_indptr[u], pe = p_indptr[u + 1];
    for (int64_t q = pb; q < pe; ++q) {
        const int i = p_indices[q];
        const float pf = p_values[q];
        const double pv = (double)(implicit ? sgn(pf) : pf);
        const int64_t e1 = s_indptr[i + 1];
        for (int64_t e = s_indptr[i] + lane; e < e1; e += 32) {
            const int s = table_insert(keys, cap, s_indices[e]);
            vals[s] = __dadd_rn(vals[s], __dmul_rn(pv, s_values[e]));
        }
        __syncwarp();
    }
    ICand* dl = lists + u * 2 * k;
    ICand* sl = dl + k;
    int64_t sb = 0, se = 0;
    if (seen_indptr) { sb = seen_indptr[u]; se = seen_indptr[u + 1]; }
    ListState st;
    int64_t nnz = 0;
    for (int t0 = 0; t0 < cap; t0 += 32) {
        const int t = t0 + lane;
        const double x = vals[t];
        const bool valid = keys[t] != kEmpty && x != 0.0;
        nnz += valid;
        offer_scores(dl, sl, k, st, x, keys[t], valid, seen_indices, sb, se, lane);
    }
    write_outputs(sl, st.cs, nnz, k, u, out_nnz, out_sparse, lane);
    write_dense_list(TableScore{keys, vals, cap}, dl, st.cd, k, n, seen_indices, sb, se, seen_indptr != nullptr,
                     out_dense + u * k, out_scores ? out_scores + u * k : nullptr, lane);
}

// Scoring, global-row path: warp `slot` takes the users with work > kHashWork at positions slot, + n_slots, ... of the
// longest-first order, accumulates each in its zeroed row of n entries in the same order as the table path, reads the
// row in column order and, after the lists, clears what the user's S rows touched.
__global__ void __launch_bounds__(256)
i2i_csr_long_kernel(int64_t n, int64_t m, const int64_t* __restrict__ s_indptr, const int32_t* __restrict__ s_indices,
                    const double* __restrict__ s_values, const int64_t* __restrict__ p_indptr,
                    const int32_t* __restrict__ p_indices, const float* __restrict__ p_values,
                    const int64_t* __restrict__ seen_indptr, const int32_t* __restrict__ seen_indices, int implicit,
                    int k, const int32_t* __restrict__ user_order, const uint64_t* __restrict__ work, int n_slots,
                    double* __restrict__ acc_rows, ICand* __restrict__ lists, int64_t* __restrict__ out_nnz,
                    int64_t* __restrict__ out_dense, int64_t* __restrict__ out_sparse, double* __restrict__ out_scores) {
    const int lane = threadIdx.x & 31;
    const int64_t slot = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (slot >= n_slots) return;
    double* row = acc_rows + slot * n;
    for (int64_t r = slot; r < m; r += n_slots) {
        const int64_t u = user_order[r];
        if (work[u] <= (uint64_t)kHashWork) break;
        const int64_t pb = p_indptr[u], pe = p_indptr[u + 1];
        for (int64_t q = pb; q < pe; ++q) {
            const int i = p_indices[q];
            const float pf = p_values[q];
            const double pv = (double)(implicit ? sgn(pf) : pf);
            const int64_t e1 = s_indptr[i + 1];
            for (int64_t e = s_indptr[i] + lane; e < e1; e += 32) {
                const int j = s_indices[e];
                row[j] = __dadd_rn(row[j], __dmul_rn(pv, s_values[e]));
            }
            __syncwarp();
        }
        ICand* dl = lists + u * 2 * k;
        ICand* sl = dl + k;
        int64_t sb = 0, se = 0;
        if (seen_indptr) { sb = seen_indptr[u]; se = seen_indptr[u + 1]; }
        ListState st;
        int64_t nnz = 0;
        for (int64_t c0 = 0; c0 < n; c0 += 32) {
            const int64_t j = c0 + lane;
            const double x = j < n ? row[j] : 0.0;
            const bool valid = x != 0.0;
            nnz += valid;
            offer_scores(dl, sl, k, st, x, (int)j, valid, seen_indices, sb, se, lane);
        }
        write_outputs(sl, st.cs, nnz, k, u, out_nnz, out_sparse, lane);
        write_dense_list(RowScore{row}, dl, st.cd, k, n, seen_indices, sb, se, seen_indptr != nullptr, out_dense + u * k,
                         out_scores ? out_scores + u * k : nullptr, lane);
        for (int64_t q = pb; q < pe; ++q) {
            const int i = p_indices[q];
            for (int64_t e = s_indptr[i] + lane; e < s_indptr[i + 1]; e += 32) row[s_indices[e]] = 0.0;
        }
        __syncwarp();
    }
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

extern "C" int pb200_cooc_build_csr(pb200_ctx* ctx, const pb200_csr_view* a, const pb200_csr_view* at, int implicit,
                                    int acc_rows, int fill, int64_t* indptr, int32_t* indices, double* values,
                                    int64_t* nnz) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, a != nullptr && at != nullptr && indptr != nullptr, "cooc_build_csr: null argument");
    PB_REQUIRE(ctx, nnz != nullptr, "cooc_build_csr: null nnz");
    PB_REQUIRE(ctx, !fill || *nnz == 0 || (indices != nullptr && values != nullptr),
               "cooc_build_csr: the fill call needs indices and values");
    const int64_t m = a->n_rows, n = a->n_cols;
    PB_REQUIRE(ctx, n > 0 && m >= 0 && n < (int64_t)2147483647 && m < (int64_t)2147483647, "cooc_build_csr: bad shape");
    PB_REQUIRE(ctx, a->n_panels == 1, "cooc_build_csr: `a` must be a plain CSR (one column panel)");
    PB_REQUIRE(ctx, at->n_rows == n && at->n_cols == m && at->nnz == a->nnz && at->n_panels == 1,
               "cooc_build_csr: `at` must be the plain CSR of A^T (pb200_csr_transpose)");
    PB_REQUIRE(ctx, acc_rows >= 1, "cooc_build_csr: acc_rows must be positive");
    if (fill && *nnz == 0) return PB200_OK;                           // nothing co-occurs: indptr is all zeros
    Scratch sc(ctx);
    uint64_t* work = nullptr;
    int32_t *iota = nullptr, *order = nullptr;
    double* acc = nullptr;
    PB_TRY(sc.alloc(&work, (size_t)n));
    PB_TRY(sc.alloc(&iota, (size_t)n));
    PB_TRY(sc.alloc(&order, (size_t)n));
    row_work_kernel<<<(unsigned)ceil_div64(n * 32, 256), 256, 0, ctx->stream>>>(at->indptr, at->indices, a->indptr, n,
                                                                               work, iota);
    PB_TRY(sort_desc(ctx, sc, work, iota, n, order));                // longest rows first
    int64_t n_long = 0;
    PB_TRY(count_long(ctx, sc, work, n, &n_long));
    const int rows = (int)std::min<int64_t>(acc_rows, n_long);        // one global row per CTA of the long-row path
    if (rows > 0) {
        PB_TRY(sc.alloc(&acc, (size_t)rows * n));
        PB_CUDA(ctx, cudaMemsetAsync(acc, 0, (size_t)rows * n * sizeof(double), ctx->stream));
    }
    const size_t smem = (size_t)kSparseWarps * kHashSlots * (sizeof(double) + sizeof(int));
    const unsigned table_grid = (unsigned)ceil_div64(n, kSparseWarps);
    if (!fill) {
        PB_CUDA(ctx, cudaMemsetAsync(indptr + n, 0, sizeof(int64_t), ctx->stream));
        PB_CUDA(ctx, cudaFuncSetAttribute(cooc_csr_table_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)smem));
        cooc_csr_table_kernel<false><<<table_grid, 32 * kSparseWarps, smem, ctx->stream>>>(
            n, a->indptr, a->indices, a->values, at->indptr, at->indices, at->values, order, work, implicit ? 1 : 0,
            indptr, nullptr, nullptr, nullptr);
        if (rows > 0)
            cooc_csr_long_kernel<false><<<rows, kLongThreads, 0, ctx->stream>>>(
                n, a->indptr, a->indices, a->values, at->indptr, at->indices, at->values, order, work, implicit ? 1 : 0,
                acc, indptr, nullptr, nullptr, nullptr);
        PB_CUDA(ctx, cudaGetLastError());
        void* temp = nullptr;                                         // row counts -> row offsets, in place
        size_t temp_bytes = 0;
        PB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, temp_bytes, indptr, indptr, n + 1, ctx->stream));
        PB_TRY(sc.alloc(reinterpret_cast<char**>(&temp), temp_bytes));
        PB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(temp, temp_bytes, indptr, indptr, n + 1, ctx->stream));
        PB_CUDA(ctx, cudaMemcpyAsync(nnz, indptr + n, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
        PB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    } else {
        PB_CUDA(ctx, cudaFuncSetAttribute(cooc_csr_table_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)smem));
        cooc_csr_table_kernel<true><<<table_grid, 32 * kSparseWarps, smem, ctx->stream>>>(
            n, a->indptr, a->indices, a->values, at->indptr, at->indices, at->values, order, work, implicit ? 1 : 0,
            nullptr, indptr, indices, values);
        if (rows > 0)
            cooc_csr_long_kernel<true><<<rows, kLongThreads, 0, ctx->stream>>>(
                n, a->indptr, a->indices, a->values, at->indptr, at->indices, at->values, order, work, implicit ? 1 : 0,
                acc, nullptr, indptr, indices, values);
        PB_CUDA(ctx, cudaGetLastError());
    }
    ctx->stats[0] += 3;
    return PB200_OK;
}

extern "C" int pb200_i2i_topk_csr(pb200_ctx* ctx, int64_t n, const int64_t* s_indptr, const int32_t* s_indices,
                                  const double* s_values, int64_t m, const int64_t* p_indptr, const int32_t* p_indices,
                                  const float* p_values, const int64_t* seen_indptr, const int32_t* seen_indices,
                                  int implicit, int k, int acc_rows, int64_t* out_nnz, int64_t* out_dense,
                                  int64_t* out_sparse, double* out_scores) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, n > 0 && m >= 0 && n < (int64_t)2147483647, "i2i_topk_csr: bad shape");
    PB_REQUIRE(ctx, k > 0 && k <= n, "i2i_topk_csr: k must be in 1..n_items");
    PB_REQUIRE(ctx, s_indptr != nullptr && p_indptr != nullptr && out_nnz != nullptr && out_dense != nullptr &&
                        out_sparse != nullptr, "i2i_topk_csr: null argument");
    PB_REQUIRE(ctx, (seen_indptr == nullptr) == (seen_indices == nullptr),
               "i2i_topk_csr: seen CSR must be both or neither");
    PB_REQUIRE(ctx, acc_rows >= 1, "i2i_topk_csr: acc_rows must be positive");
    if (m == 0) return PB200_OK;
    PB_REQUIRE(ctx, m < (int64_t)2147483647, "i2i_topk_csr: too many users");
    Scratch sc(ctx);
    uint64_t* work = nullptr;
    int32_t *iota = nullptr, *order = nullptr;
    ICand* lists = nullptr;
    double* acc = nullptr;
    PB_TRY(sc.alloc(&work, (size_t)m));
    PB_TRY(sc.alloc(&iota, (size_t)m));
    PB_TRY(sc.alloc(&order, (size_t)m));
    PB_TRY(sc.alloc(&lists, (size_t)m * 2 * k));
    // work of a user: the nonzeros of its S rows (the products that form its scores)
    row_work_kernel<<<(unsigned)ceil_div64(m * 32, 256), 256, 0, ctx->stream>>>(p_indptr, p_indices, s_indptr, m, work,
                                                                               iota);
    PB_TRY(sort_desc(ctx, sc, work, iota, m, order));                 // most work first
    int64_t n_long = 0;
    PB_TRY(count_long(ctx, sc, work, m, &n_long));
    const int rows = (int)std::min<int64_t>(acc_rows, n_long);        // one global row per warp of the long-user path
    if (rows > 0) {
        PB_TRY(sc.alloc(&acc, (size_t)rows * n));
        PB_CUDA(ctx, cudaMemsetAsync(acc, 0, (size_t)rows * n * sizeof(double), ctx->stream));
    }
    const size_t smem = (size_t)kSparseWarps * kHashSlots * (sizeof(double) + sizeof(int));
    PB_CUDA(ctx, cudaFuncSetAttribute(i2i_csr_table_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (rows > 0)
        i2i_csr_long_kernel<<<(unsigned)ceil_div64((int64_t)rows * 32, 256), 256, 0, ctx->stream>>>(
            n, m, s_indptr, s_indices, s_values, p_indptr, p_indices, p_values, seen_indptr, seen_indices,
            implicit ? 1 : 0, k, order, work, rows, acc, lists, out_nnz, out_dense, out_sparse, out_scores);
    i2i_csr_table_kernel<<<(unsigned)ceil_div64(m, kSparseWarps), 32 * kSparseWarps, smem, ctx->stream>>>(
        n, m, s_indptr, s_indices, s_values, p_indptr, p_indices, p_values, seen_indptr, seen_indices, implicit ? 1 : 0,
        k, order, work, lists, out_nnz, out_dense, out_sparse, out_scores);
    ctx->stats[0] += 3;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

// Top-k and seen-item handling for a caller's DENSE score block (scores that did not come from our factors):
//   pb200_topk_dense      RecommenderModel.get_topk_elements, dense branch (polara/recommender/models.py:561-563,
//                         topsort 488-491), optionally fused with the seen-item handling so that one pass suffices;
//   pb200_downvote_dense  RecommenderModel.downvote_seen_items, dense branch (models.py:510-519): in place,
//                         S[row, col] <- min(S) - (max(S_seen) - S[row, col]) - 1 for the seen pairs.
// One warp per row streams the row once (coalesced), keeps the running top-k in a sorted list (threshold filter +
// warp-cooperative insertion); HBM-bound on m * n * sizeof(score).  Order: (score desc, id asc) -- the reference leaves
// ties unspecified (argpartition), NaN scores are not supported (they never enter a list).
#include "common.cuh"

#include <math_constants.h>

namespace {

template <typename T>
struct DCand { T score; int32_t id; };

template <typename T> __device__ __forceinline__ T neg_inf();
template <> __device__ __forceinline__ float neg_inf<float>() { return -CUDART_INF_F; }
template <> __device__ __forceinline__ double neg_inf<double>() { return -CUDART_INF; }

template <typename T>
__device__ __forceinline__ bool before(T sa, int ia, T sb, int ib) { return sa > sb || (sa == sb && ia < ib); }

// warp-cooperative insertion into a sorted list of capacity cap (fill cnt, uniform); returns the new fill
template <typename T>
__device__ __forceinline__ int list_insert(DCand<T>* list, int cap, int cnt, T s, int id, int lane) {
    if (cap <= 0) return cnt;
    if (cnt == cap) {
        DCand<T> last = list[cap - 1];
        if (!before(s, id, last.score, last.id)) return cnt;
    }
    int pos = 0;
    for (int base = 0; base < cnt; base += 32) {
        int i = base + lane;
        bool b = false;
        if (i < cnt) { DCand<T> c = list[i]; b = before(c.score, c.id, s, id); }
        pos += __popc(__ballot_sync(0xffffffffu, b));
    }
    const int last_dst = min(cnt, cap - 1);
    for (int hi = last_dst; hi > pos; hi -= 32) {
        int dst = hi - lane;
        DCand<T> c;
        bool act = dst > pos;
        if (act) c = list[dst - 1];
        __syncwarp();
        if (act) list[dst] = c;
        __syncwarp();
    }
    if (lane == 0) { DCand<T> c; c.score = s; c.id = id; list[pos] = c; }
    __syncwarp();
    return min(cnt + 1, cap);
}

__device__ __forceinline__ bool in_sorted(const int32_t* __restrict__ a, int64_t beg, int64_t end, int key) {
    int64_t lo = beg, hi = end;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (__ldg(a + mid) < key) lo = mid + 1; else hi = mid;
    }
    return lo < end && __ldg(a + lo) == key;
}

template <typename T>
__global__ void __launch_bounds__(256)
topk_dense_kernel(const T* __restrict__ S, int64_t lds, int64_t m, int64_t n, const int64_t* __restrict__ seen_indptr,
                  const int32_t* __restrict__ seen_indices, int k, DCand<T>* __restrict__ lists,
                  int64_t* __restrict__ out_ids, T* __restrict__ out_scores) {
    const int lane = threadIdx.x & 31;
    const int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (u >= m) return;
    DCand<T>* list = lists + u * k;
    const T* row = S + u * lds;
    int64_t sb = 0, se = 0;
    if (seen_indptr) { sb = seen_indptr[u]; se = seen_indptr[u + 1]; }
    int cnt = 0;
    T thr = neg_inf<T>();
    for (int64_t base = 0; base < n; base += 32) {
        const int64_t j = base + lane;
        T x = neg_inf<T>();
        bool pass = false;
        if (j < n) {
            x = row[j];
            // ids ascend along the scan: an equal score later in the row never displaces an earlier one
            pass = (cnt < k) ? (x == x) : (x > thr);
            if (pass && sb < se) pass = !in_sorted(seen_indices, sb, se, (int)j);
        }
        unsigned mask = __ballot_sync(0xffffffffu, pass);
        while (mask) {
            const int t = __ffs(mask) - 1;
            mask &= mask - 1;
            const T xs = __shfl_sync(0xffffffffu, x, t);
            cnt = list_insert(list, k, cnt, xs, (int)(base + t), lane);
            if (cnt == k) thr = list[k - 1].score;
        }
    }
    // fewer than k unseen items: the seen ones follow by (score desc, id asc) -- the order the pushed-down scores of
    // downvote_seen_items keep (models.py:517-519)
    if (cnt < k && sb < se) {
        DCand<T>* tail = list + cnt;
        const int cap = k - cnt;
        int tc = 0;
        for (int64_t p0 = sb; p0 < se; p0 += 32) {
            const int64_t p = p0 + lane;
            int id = -1;
            T x = neg_inf<T>();
            if (p < se) { id = __ldg(seen_indices + p); if (id >= 0 && id < n) x = row[id]; else id = -1; }
            unsigned mask = __ballot_sync(0xffffffffu, id >= 0 && x == x);
            while (mask) {
                const int t = __ffs(mask) - 1;
                mask &= mask - 1;
                tc = list_insert(tail, cap, tc, __shfl_sync(0xffffffffu, x, t), __shfl_sync(0xffffffffu, id, t), lane);
            }
        }
        cnt += tc;
    }
    __syncwarp();
    for (int i = lane; i < k; i += 32) {
        const bool ok = i < cnt;
        out_ids[u * k + i] = ok ? (int64_t)list[i].id : -1;          // the reference pads with -1 (models.py:73)
        if (out_scores) out_scores[u * k + i] = ok ? list[i].score : neg_inf<T>();
    }
}

// ---- downvote_seen_items, dense branch ------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
minmax_partial_kernel(const T* __restrict__ S, int64_t lds, int64_t m, int64_t n, const int64_t* __restrict__ rows,
                      const int64_t* __restrict__ cols, int64_t nnz, double* __restrict__ partial /*[grid][2]*/) {
    double mn = CUDART_INF, mx = -CUDART_INF;
    const int64_t total = m * n, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const double x = (double)S[(i / n) * lds + i % n];
        mn = fmin(mn, x);
    }
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += stride)
        mx = fmax(mx, (double)S[rows[i] * lds + cols[i]]);
    __shared__ double smn[256], smx[256];
    smn[threadIdx.x] = mn; smx[threadIdx.x] = mx;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) { smn[threadIdx.x] = fmin(smn[threadIdx.x], smn[threadIdx.x + o]); smx[threadIdx.x] = fmax(smx[threadIdx.x], smx[threadIdx.x + o]); }
        __syncthreads();
    }
    if (threadIdx.x == 0) { partial[2 * blockIdx.x] = smn[0]; partial[2 * blockIdx.x + 1] = smx[0]; }
}

__global__ void minmax_final_kernel(const double* __restrict__ partial, int nblk, double* __restrict__ out2) {
    double mn = CUDART_INF, mx = -CUDART_INF;
    for (int i = threadIdx.x; i < nblk; i += blockDim.x) { mn = fmin(mn, partial[2 * i]); mx = fmax(mx, partial[2 * i + 1]); }
    __shared__ double smn[256], smx[256];
    smn[threadIdx.x] = mn; smx[threadIdx.x] = mx;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) { smn[threadIdx.x] = fmin(smn[threadIdx.x], smn[threadIdx.x + o]); smx[threadIdx.x] = fmax(smx[threadIdx.x], smx[threadIdx.x + o]); }
        __syncthreads();
    }
    if (threadIdx.x == 0) { out2[0] = smn[0]; out2[1] = smx[0]; }
}

// new values are computed from the ORIGINAL seen scores (the reference gathers them all before it writes, and repeated
// coordinates are idempotent): gather first, write after
// min(S) - (max(S_seen) - x) - 1 in the dtype of the scores, one rounding per operation as numpy evaluates it.  mn and
// mx are elements of S, so narrowing them back to float is exact; __fsub_rn keeps the three float32 steps apart.
__device__ __forceinline__ float downvote_value(double mn, double mx, float x) {
    return __fsub_rn(__fsub_rn((float)mn, __fsub_rn((float)mx, x)), 1.0f);
}
__device__ __forceinline__ double downvote_value(double mn, double mx, double x) { return mn - (mx - x) - 1.0; }

template <typename T>
__global__ void downvote_gather_kernel(const T* __restrict__ S, int64_t lds, const int64_t* __restrict__ rows,
                                       const int64_t* __restrict__ cols, int64_t nnz, const double* __restrict__ mm,
                                       T* __restrict__ lowered) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += stride)
        lowered[i] = downvote_value(mm[0], mm[1], S[rows[i] * lds + cols[i]]);
}
template <typename T>
__global__ void downvote_scatter_kernel(T* __restrict__ S, int64_t lds, const int64_t* __restrict__ rows,
                                        const int64_t* __restrict__ cols, int64_t nnz, const T* __restrict__ lowered) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += stride) S[rows[i] * lds + cols[i]] = lowered[i];
}

template <typename T>
int topk_dense_impl(pb200_ctx* ctx, const T* S, int64_t lds, int64_t m, int64_t n, const int64_t* seen_indptr,
                    const int32_t* seen_indices, int k, int64_t* out_ids, T* out_scores) {
    Scratch sc(ctx);
    DCand<T>* lists = nullptr;
    PB_TRY(sc.alloc(&lists, (size_t)m * k));
    topk_dense_kernel<T><<<(unsigned)ceil_div64(m * 32, 256), 256, 0, ctx->stream>>>(S, lds, m, n, seen_indptr, seen_indices, k,
                                                                                   lists, out_ids, out_scores);
    ctx->stats[0] += 1;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

template <typename T>
int downvote_impl(pb200_ctx* ctx, T* S, int64_t lds, int64_t m, int64_t n, const int64_t* rows, const int64_t* cols, int64_t nnz) {
    Scratch sc(ctx);
    const int nblk = 4 * ctx->num_sms;
    double *partial = nullptr, *mm = nullptr;
    T* lowered = nullptr;
    PB_TRY(sc.alloc(&partial, (size_t)2 * nblk));
    PB_TRY(sc.alloc(&mm, 2));
    PB_TRY(sc.alloc(&lowered, (size_t)nnz));
    minmax_partial_kernel<T><<<nblk, 256, 0, ctx->stream>>>(S, lds, m, n, rows, cols, nnz, partial);
    minmax_final_kernel<<<1, 256, 0, ctx->stream>>>(partial, nblk, mm);
    downvote_gather_kernel<T><<<nblk, 256, 0, ctx->stream>>>(S, lds, rows, cols, nnz, mm, lowered);
    downvote_scatter_kernel<T><<<nblk, 256, 0, ctx->stream>>>(S, lds, rows, cols, nnz, lowered);
    ctx->stats[0] += 4;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

}  // namespace

extern "C" int pb200_topk_dense(pb200_ctx* ctx, const void* S, int dtype, int64_t lds, int64_t m, int64_t n,
                                const int64_t* seen_indptr, const int32_t* seen_indices, int k, int64_t* out_ids,
                                void* out_scores) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, dtype == PB200_F32 || dtype == PB200_F64, "topk_dense: scores must be f32 or f64");
    PB_REQUIRE(ctx, m >= 0 && n > 0 && lds >= n && n < (int64_t)2147483647, "topk_dense: bad shape");
    PB_REQUIRE(ctx, k > 0 && k <= n, "topk_dense: k must be in 1..n");          // np.argpartition raises for k > n
    PB_REQUIRE(ctx, S != nullptr && out_ids != nullptr, "topk_dense: null argument");
    PB_REQUIRE(ctx, (seen_indptr == nullptr) == (seen_indices == nullptr), "topk_dense: seen CSR must be both or neither");
    if (m == 0) return PB200_OK;
    if (dtype == PB200_F32)
        return topk_dense_impl<float>(ctx, static_cast<const float*>(S), lds, m, n, seen_indptr, seen_indices, k, out_ids,
                                      static_cast<float*>(out_scores));
    return topk_dense_impl<double>(ctx, static_cast<const double*>(S), lds, m, n, seen_indptr, seen_indices, k, out_ids,
                                   static_cast<double*>(out_scores));
}

extern "C" int pb200_downvote_dense(pb200_ctx* ctx, void* S, int dtype, int64_t lds, int64_t m, int64_t n,
                                    const int64_t* rows, const int64_t* cols, int64_t nnz) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, dtype == PB200_F32 || dtype == PB200_F64, "downvote_dense: scores must be f32 or f64");
    PB_REQUIRE(ctx, m > 0 && n > 0 && lds >= n && S != nullptr, "downvote_dense: bad shape");
    if (nnz == 0) return PB200_OK;
    PB_REQUIRE(ctx, rows != nullptr && cols != nullptr, "downvote_dense: null index arrays");
    if (dtype == PB200_F32) return downvote_impl<float>(ctx, static_cast<float*>(S), lds, m, n, rows, cols, nnz);
    return downvote_impl<double>(ctx, static_cast<double*>(S), lds, m, n, rows, cols, nnz);
}

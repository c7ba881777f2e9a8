// C-ABI entry points that are not tied to one kernel file: context, scoring front end.
#include <algorithm>
#include <cstdlib>

#include "topk_common.cuh"

namespace {

__global__ void __launch_bounds__(256)
score_dense_kernel(const float* __restrict__ E, int64_t lde, const float* __restrict__ V, int64_t ldv,
                   int64_t m, int64_t n, int r, float* __restrict__ S, int64_t lds) {
    // one warp per item, all (few) users: canonical fp32 score
    const int lane = threadIdx.x & 31;
    int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (j >= n) return;
    for (int64_t u = lane; u < m; u += 32) S[u * lds + j] = exact_score(E + u * lde, V + j * ldv, r);
}

// out[a] = canonical fp32 score of (user uidx[a], item iidx[a]): sampled evaluation (inner_product_at,
// polara/lib/sparse.py:58-72) -- one thread per pair, the user's row stays in L1 across its width consecutive pairs
__global__ void gather_dot_kernel(const float* __restrict__ E, int64_t lde, const float* __restrict__ V, int64_t ldv, int r,
                                  const int64_t* __restrict__ uidx, const int64_t* __restrict__ iidx, int64_t count,
                                  int64_t m, int64_t n, float* __restrict__ out) {
    int64_t a = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; a < count; a += stride) {
        const int64_t u = uidx[a], j = iidx[a];
        out[a] = (u >= 0 && u < m && j >= 0 && j < n) ? exact_score(E + u * lde, V + j * ldv, r) : CUDART_NAN_F;
    }
}

}  // namespace

extern "C" int pb200_version(void) { return 100; }

extern "C" int pb200_ctx_create(int device, void* stream, pb200_ctx** out) {
    if (!out) return PB200_EINVAL;
    *out = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || device < 0 || device >= count) return PB200_ECUDA;
    if (cudaSetDevice(device) != cudaSuccess) return PB200_ECUDA;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return PB200_ECUDA;
    pb200_ctx* ctx = new pb200_ctx();
    ctx->device = device;
    ctx->stream = static_cast<cudaStream_t>(stream);
    ctx->num_sms = prop.multiProcessorCount;
    // profiling aid: PB200_PRUNE=0 starts the context with the early termination of the scoring sweep off (same as
    // pb200_set_prune(ctx, 0)); results are identical either way
    if (const char* e = getenv("PB200_PRUNE")) ctx->prune = atoi(e) != 0;
    if (prop.major != 9 || prop.minor != 0) {
        // built for sm_90a only: refuse loudly rather than fail at the first launch
        delete ctx;
        return PB200_ENOTIMPL;
    }
    {
        // scratch buffers come from the stream-ordered pool; keep freed blocks cached across synchronisations
        // (the default threshold 0 hands them back to the driver at every sync, and re-allocating them is slow)
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
            uint64_t keep = UINT64_MAX;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
    }
    if (cudaMalloc(&ctx->d_stats, 8 * sizeof(uint64_t)) != cudaSuccess) { delete ctx; return PB200_ENOMEM; }
    cudaMemset(ctx->d_stats, 0, 8 * sizeof(uint64_t));
    if (cudaHostAlloc(&ctx->h_dbg, 16 * sizeof(unsigned long long), cudaHostAllocMapped) == cudaSuccess) memset(ctx->h_dbg, 0, 16 * sizeof(unsigned long long)); else ctx->h_dbg = nullptr;
    cudaEventCreate(&ctx->ev0);
    cudaEventCreate(&ctx->ev1);
    *out = ctx;
    return PB200_OK;
}

extern "C" int pb200_ctx_destroy(pb200_ctx* ctx) {
    if (!ctx) return PB200_OK;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    cudaFree(ctx->d_stats);
    if (ctx->h_dbg) cudaFreeHost(ctx->h_dbg);
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    delete ctx;
    return PB200_OK;
}

extern "C" const char* pb200_last_error(pb200_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

extern "C" int pb200_debug_dump(pb200_ctx* ctx) {
    if (!ctx || !ctx->h_dbg) return PB200_EINVAL;
    fprintf(stderr, "pb200 debug:");
    for (int i = 0; i < 8; ++i) fprintf(stderr, " %llx", ctx->h_dbg[i]);
    fprintf(stderr, "\n");
    return PB200_OK;
}

extern "C" int pb200_ctx_sync(pb200_ctx* ctx) {
    PB_ENTER(ctx);
    PB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return PB200_OK;
}

extern "C" int pb200_ctx_set_stream(pb200_ctx* ctx, void* stream) {
    if (!ctx) return PB200_EINVAL;
    ctx->stream = static_cast<cudaStream_t>(stream);
    return PB200_OK;
}

extern "C" int pb200_set_score_kernel(pb200_ctx* ctx, int kind) {
    if (!ctx) return PB200_EINVAL;
    PB_REQUIRE(ctx, kind == 0 || kind == 1, "score kernel must be 0 (simt) or 1 (tc: wgmma filter + exact rescoring)");
    ctx->score_kernel = kind;
    return PB200_OK;
}

extern "C" int pb200_set_spmm_kernel(pb200_ctx* ctx, int kind) {
    if (!ctx) return PB200_EINVAL;
    PB_REQUIRE(ctx, kind >= 0 && kind <= 4, "spmm kernel must be 0 (row-owned gathers), 1 (staged by cp.async.bulk), 2 (staged by cp.async), 3 (nnz windows, 128-bit gathers) or 4 (nnz windows, 32-bit gathers)");
    ctx->spmm_kernel = kind;
    return PB200_OK;
}

extern "C" int pb200_set_prune(pb200_ctx* ctx, int on) {
    if (!ctx) return PB200_EINVAL;
    ctx->prune = on ? 1 : 0;
    return PB200_OK;
}

extern "C" int pb200_set_reduce_hook(pb200_ctx* ctx, pb200_reduce_fn fn, void* user) {
    if (!ctx) return PB200_EINVAL;
    ctx->reduce_fn = fn;
    ctx->reduce_user = user;
    return PB200_OK;
}

extern "C" int pb200_set_bound_hook(pb200_ctx* ctx, pb200_reduce_fn fn, void* user) {
    if (!ctx) return PB200_EINVAL;
    ctx->bound_fn = fn;
    ctx->bound_user = user;
    return PB200_OK;
}

extern "C" int pb200_get_stats(pb200_ctx* ctx, uint64_t* out8_host) {
    if (!out8_host) return PB200_EINVAL;
    PB_ENTER(ctx);
    uint64_t dev[8];
    PB_CUDA(ctx, cudaMemcpyAsync(dev, ctx->d_stats, sizeof dev, cudaMemcpyDeviceToHost, ctx->stream));
    PB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < 8; ++i) out8_host[i] = ctx->stats[i] + dev[i];
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1) == cudaSuccess) out8_host[4] = (uint64_t)(ms * 1000.0f);
    else { cudaGetLastError(); out8_host[4] = 0; }
    return PB200_OK;
}

static int score_front(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv, int64_t m,
                       int64_t n, int r, const int64_t* seen_indptr, const int32_t* seen_indices, int k,
                       int64_t item_offset, int64_t* out_ids, float* out_scores, pb200_cand* out_cands) {
    PB_REQUIRE(ctx, m >= 0 && n > 0 && r > 0, "score_topk: bad shape");
    PB_REQUIRE(ctx, k > 0 && k <= 1024, "score_topk: k must be in 1..1024");
    PB_REQUIRE(ctx, lde >= r && ldv >= r, "score_topk: leading dimension smaller than rank");
    PB_REQUIRE(ctx, (seen_indptr == nullptr) == (seen_indices == nullptr), "score_topk: seen CSR must be both or neither");
    PB_REQUIRE(ctx, n < (int64_t)2147483647, "score_topk: item count must fit int32");
    if (m == 0) return PB200_OK;
    Scratch sc(ctx);
    pb200_cand* lists = nullptr;
    int parts = 1;
    bool use_tc = ctx->score_kernel == 1;
    if (use_tc) {
        // ranks whose padded K does not leave two pipeline stages in shared memory (r > ~250) are not implemented on the
        // tensor-core path: the exact CUDA-core kernel takes them (same results by construction)
        int st = pb_score_tc(ctx, E, lde, V, ldv, m, n, r, seen_indptr, seen_indices, item_offset, k, &parts, &lists, sc);
        if (st == PB200_ENOTIMPL) { use_tc = false; ctx->err.clear(); }
        else PB_TRY(st);
    }
    if (!use_tc) {
        int64_t user_tiles = ceil_div64(m, 64), item_tiles = ceil_div64(n, 128);
        int64_t want = ceil_div64(4 * (int64_t)ctx->num_sms, user_tiles);
        parts = (int)std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>(want, 32), item_tiles));
        PB_TRY(sc.alloc(&lists, (size_t)parts * m * k));
        PB_TRY(pb_score_simt(ctx, E, lde, V, ldv, m, n, r, seen_indptr, seen_indices, item_offset, k, parts, lists));
    }
    // the seen fill-up needs E,V of the whole item range: only offered for unsharded calls
    bool fill = out_cands == nullptr;
    PB_TRY(pb_merge_lists(ctx, lists, parts, m * (int64_t)k, m, k, item_offset, out_ids, out_scores, out_cands,
                          fill ? E : nullptr, lde, fill ? V : nullptr, ldv, r, n, seen_indptr, seen_indices));
    return PB200_OK;
}

extern "C" int pb200_score_topk(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv,
                                int64_t m, int64_t n, int r, const int64_t* seen_indptr,
                                const int32_t* seen_indices, int k, int64_t item_offset, int64_t* out_ids,
                                float* out_scores) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, out_ids != nullptr, "score_topk: out_ids is required");
    return score_front(ctx, E, lde, V, ldv, m, n, r, seen_indptr, seen_indices, k, item_offset, out_ids,
                       out_scores, nullptr);
}

extern "C" int pb200_score_topk_cands(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv,
                                      int64_t m, int64_t n, int r, const int64_t* seen_indptr,
                                      const int32_t* seen_indices, int k, int64_t item_offset,
                                      pb200_cand* out_cands) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, out_cands != nullptr, "score_topk_cands: out_cands is required");
    PB_REQUIRE(ctx, item_offset + n < (int64_t)2147483647, "score_topk_cands: global item id must fit int32");
    return score_front(ctx, E, lde, V, ldv, m, n, r, seen_indptr, seen_indices, k, item_offset, nullptr, nullptr,
                       out_cands);
}

extern "C" int pb200_merge_cands(pb200_ctx* ctx, const pb200_cand* in, int parts, int64_t m, int k,
                                 int64_t* out_ids, float* out_scores) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, out_ids != nullptr && k > 0, "merge_cands: bad arguments");
    return pb_merge_lists(ctx, in, parts, m * (int64_t)k, m, k, 0, out_ids, out_scores, nullptr, nullptr, 0,
                          nullptr, 0, 0, 0, nullptr, nullptr);
}

extern "C" int pb200_merge_cands_fill(pb200_ctx* ctx, const pb200_cand* in, int parts, int64_t part_stride, int64_t m, int k,
                                      const float* E, int64_t lde, const float* V, int64_t ldv, int r, int64_t n,
                                      const int64_t* seen_indptr, const int32_t* seen_indices,
                                      int64_t* out_ids, float* out_scores) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, out_ids != nullptr && k > 0 && part_stride >= m * (int64_t)k, "merge_cands_fill: bad arguments");
    PB_REQUIRE(ctx, E && V && seen_indptr && seen_indices && lde >= r && ldv >= r, "merge_cands_fill: factors and seen lists are required");
    return pb_merge_lists(ctx, in, parts, part_stride, m, k, 0, out_ids, out_scores, nullptr, E, lde, V, ldv, r, n,
                          seen_indptr, seen_indices);
}

extern "C" int pb200_gather_dot(pb200_ctx* ctx, const float* E, int64_t lde, int64_t m, const float* V, int64_t ldv, int64_t n,
                                int r, const int64_t* user_idx, const int64_t* item_idx, int64_t count, float* out) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, r > 0 && lde >= r && ldv >= r && count >= 0, "gather_dot: bad shape");
    if (count == 0) return PB200_OK;
    PB_REQUIRE(ctx, E && V && user_idx && item_idx && out, "gather_dot: null argument");
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div64(count, 256), 16 * (int64_t)ctx->num_sms);
    gather_dot_kernel<<<blocks, 256, 0, ctx->stream>>>(E, lde, V, ldv, r, user_idx, item_idx, count, m, n, out);
    ctx->stats[0] += 1;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

extern "C" int pb200_score_dense(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv,
                                 int64_t m, int64_t n, int r, float* S, int64_t lds) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, lds >= n && lde >= r && ldv >= r, "score_dense: leading dimension too small");
    if (m == 0 || n == 0) return PB200_OK;
    score_dense_kernel<<<(unsigned)ceil_div64(n * 32, 256), 256, 0, ctx->stream>>>(E, lde, V, ldv, m, n, r, S, lds);
    ctx->stats[0] += 1;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

// Shared plumbing for the polara_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/polara_b200.h"

struct pb200_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    int num_sms = 132;
    int score_kernel = 1;          // 0 = SIMT exact, 1 = tensor-core (wgmma) filter + exact rescoring
    int spmm_kernel = 3;           // 3 = nnz windows + register gathers (default), 1 / 2 = X rows staged in shared memory by
                                   // cp.async.bulk / cp.async, 0 = row-owned register gathers (round-1 kernel)
    int prune = 1;                 // 1 = stop a user tile's sweep where ||e|| * ||v|| can no longer reach its threshold
    std::string err;
    uint64_t stats[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint64_t* d_stats = nullptr;   // device counters (8 x u64)
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // bracket the last fused scoring kernel
    unsigned long long* h_dbg = nullptr;        // pinned, device-mapped: survives a trapped kernel (timeout diagnostics)
    pb200_reduce_fn reduce_fn = nullptr;        // row-sharded build: global sum of partial results (pb200_set_reduce_hook)
    void* reduce_user = nullptr;
    pb200_reduce_fn bound_fn = nullptr;         // item-sharded scoring: elementwise MAX of the seed bounds over the shards
    void* bound_user = nullptr;
    int sampler_map_slots = 3072;               // position-map slots per warp in shared memory (pb200_set_sampler_map_slots)
    uint64_t sampler_stats[4] = {0, 0, 0, 0};   // last sampler call: users on the shared / global map path, global slots, launches
};

#define PB_CUDA(ctx, call)                                                              \
    do {                                                                                \
        cudaError_t e__ = (call);                                                       \
        if (e__ != cudaSuccess) {                                                       \
            char b__[512];                                                              \
            snprintf(b__, sizeof b__, "%s:%d %s -> %s", __FILE__, __LINE__, #call,      \
                     cudaGetErrorString(e__));                                          \
            (ctx)->err = b__;                                                           \
            return e__ == cudaErrorMemoryAllocation ? PB200_ENOMEM : PB200_ECUDA;       \
        }                                                                               \
    } while (0)

// every C-ABI entry point starts with this: null check + make the context's device current (a process may hold one
// context per device; kernels and attributes are per device)
#define PB_ENTER(ctx)                                                                   \
    do {                                                                                \
        if (!(ctx)) return PB200_EINVAL;                                                \
        if (cudaSetDevice((ctx)->device) != cudaSuccess) {                              \
            (ctx)->err = "cudaSetDevice failed";                                        \
            return PB200_ECUDA;                                                         \
        }                                                                               \
    } while (0)

#define PB_REQUIRE(ctx, cond, msg)                                                      \
    do {                                                                                \
        if (!(cond)) {                                                                  \
            (ctx)->err = std::string("invalid argument: ") + (msg);                     \
            return PB200_EINVAL;                                                        \
        }                                                                               \
    } while (0)

#define PB_TRY(expr)                                                                    \
    do {                                                                                \
        int s__ = (expr);                                                               \
        if (s__ != PB200_OK) return s__;                                                \
    } while (0)

// Stream-ordered scratch memory, released when the guard leaves scope.
struct Scratch {
    pb200_ctx* ctx;
    std::vector<void*> ptrs;
    explicit Scratch(pb200_ctx* c) : ctx(c) {}
    ~Scratch() {
        for (void* p : ptrs) cudaFreeAsync(p, ctx->stream);
    }
    template <typename T>
    int alloc(T** out, size_t count) {
        void* p = nullptr;
        size_t bytes = count * sizeof(T);
        if (bytes == 0) bytes = sizeof(T);
        cudaError_t e = cudaMallocAsync(&p, bytes, ctx->stream);
        if (e != cudaSuccess) {
            char b[256];
            snprintf(b, sizeof b, "cudaMallocAsync(%zu bytes) -> %s", bytes, cudaGetErrorString(e));
            ctx->err = b;
            cudaGetLastError();
            *out = nullptr;
            return PB200_ENOMEM;
        }
        ptrs.push_back(p);
        *out = static_cast<T*>(p);
        return PB200_OK;
    }
};

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Sum a device buffer over all row shards through the caller's hook (no-op when the matrix is not sharded).
static inline int pb_reduce(pb200_ctx* ctx, void* dev_ptr, int64_t count, int dtype) {
    if (!ctx->reduce_fn) return PB200_OK;
    int st = ctx->reduce_fn(ctx->reduce_user, dev_ptr, count, dtype);
    if (st != 0) {
        ctx->err = "reduce hook failed with status " + std::to_string(st);
        return PB200_ECUDA;
    }
    return PB200_OK;
}

// ---- internal entry points shared between translation units -----------------------
int pb_gram(pb200_ctx* ctx, const float* Y, int64_t n, int c, int64_t ld, double* G /*[c x c]*/);
// eigen-decomposition of symmetric PSD G [c x c] (destroyed); lam [c] descending,
// vecs [c x c] row i = eigenvector i (matching lam[i]).
int pb_eig_psd(pb200_ctx* ctx, double* G, int c, double* lam, double* vecs);
// C[n x c2] = Y[n x c] * W[c x c2]   (W float32 row-major, ldw)
int pb_right_multiply(pb200_ctx* ctx, const float* Y, int64_t n, int c, int64_t ldy,
                      const float* W, int c2, int64_t ldw, float* C, int64_t ldc);
int pb_fill_gaussian(pb200_ctx* ctx, float* X, int64_t count, uint64_t seed);
// orthonormalise columns of Y [n x c] into Q (SVQB: Q = Y W L^-1/2); lam_out (device,
// c doubles, descending eigenvalues of Y^T Y) may be nullptr.  rows_sharded: Y holds this shard's rows only,
// the Gram matrix is summed over the shards (pb_reduce) before the eigen-decomposition.
int pb_orthonormalize(pb200_ctx* ctx, const float* Y, int64_t n, int c, int64_t ldy, float* Q,
                      int64_t ldq, double* lam_out, bool rows_sharded = false);
int pb_spmm_impl(pb200_ctx* ctx, int64_t n_rows, int64_t nnz, const int64_t* indptr,
                 const int32_t* indices, const float* values, const float* X, int64_t ldx,
                 float* Y, int64_t ldy, int ell);
// same for a (possibly panel-major) matrix view
int pb_spmm_view(pb200_ctx* ctx, const pb200_csr_view* a, const float* X, int64_t ldx, float* Y, int64_t ldy, int ell);
// C[ca x cb] = A^T B for two tall panels with the same row count (fp64 accumulation, deterministic)
int pb_cross_gram(pb200_ctx* ctx, const float* A, int ca, int64_t lda, const float* B, int cb, int64_t ldb, int64_t n,
                  double* C /*[ca x cb]*/);

int pb_score_simt(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv,
                  int64_t m, int64_t n, int r, const int64_t* seen_indptr,
                  const int32_t* seen_indices, int64_t seen_offset, int k, int parts, pb200_cand* lists,
                  const int32_t* id_map = nullptr);
int pb_score_tc(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv,
                int64_t m, int64_t n, int r, const int64_t* seen_indptr,
                const int32_t* seen_indices, int64_t seen_offset, int k, int* parts_out,
                pb200_cand** lists_out, Scratch& scratch);
int pb_merge_lists(pb200_ctx* ctx, const pb200_cand* lists, int parts, int64_t part_stride,
                   int64_t m, int k, int64_t item_offset, int64_t* out_ids, float* out_scores,
                   pb200_cand* out_cands,
                   // optional fill-up with seen items when fewer than k unseen exist
                   const float* E, int64_t lde, const float* V, int64_t ldv, int r, int64_t n,
                   const int64_t* seen_indptr, const int32_t* seen_indices);

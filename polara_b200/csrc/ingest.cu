// Device-side ingest: COO triplets (as RecommenderData.to_coo / test_to_coo hand them over: int64 indices, float64 or
// float32 feedback; polara/recommender/data.py:794-817, 835-862) -> the CSR the kernels read (indptr int64, indices
// int32 sorted within a row, values float32, duplicates summed).  Replaces scipy's coo_matrix(...).tocsr()
// (polara/recommender/models.py:169-174) and csr_matrix((fdbk, (user, item))) (models.py:208-210), including the
// "drop zero feedback" filter of get_test_matrix (models.py:197-201).
//
// Input that is already strictly increasing in (row, col) -- what a data model sorted by user and item yields, and what
// the benchmark feeds -- takes the fast path: one checking pass, a dtype conversion and a row-pointer search.  Anything
// else goes through a stable radix sort of the 64-bit keys row * n_cols + col (CUB; format conversion only) and a
// segmented sum of duplicates in input order (deterministic).
#include <algorithm>
#include <cmath>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace {

__device__ __forceinline__ double load_val(const void* vals, int dtype, int64_t i) {
    if (!vals) return 1.0;
    return dtype == PB200_F64 ? reinterpret_cast<const double*>(vals)[i] : (double)reinterpret_cast<const float*>(vals)[i];
}

// flags[0] |= 1 if some (row, col) is not strictly greater than its predecessor; |= 2 if an index is out of range;
// |= 4 if a zero value has to be dropped; |= 8 if the ROWS decrease somewhere
__global__ void coo_check_kernel(const int64_t* __restrict__ rows, int64_t rs, const int64_t* __restrict__ cols, int64_t cs,
                                 const void* __restrict__ vals, int dtype, int drop_zeros, int64_t nnz, int64_t n_rows,
                                 int64_t n_cols, int* __restrict__ flags) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int f = 0;
    for (; i < nnz; i += stride) {
        const int64_t r = rows[i * rs], c = cols[i * cs];
        if (r < 0 || r >= n_rows || c < 0 || c >= n_cols) f |= 2;
        if (i > 0) {
            const int64_t pr = rows[(i - 1) * rs], pc = cols[(i - 1) * cs];
            if (pr > r || (pr == r && pc >= c)) f |= 1;
            if (pr > r) f |= 8;
        }
        if (drop_zeros && load_val(vals, dtype, i) == 0.0) f |= 4;
    }
    if (f) atomicOr(flags, f);
}

__global__ void coo_convert_sorted_kernel(const int64_t* __restrict__ cols, int64_t cs, const void* __restrict__ vals,
                                          int dtype, int64_t nnz, int32_t* __restrict__ indices, float* __restrict__ values) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < nnz; i += stride) { indices[i] = (int32_t)cols[i * cs]; values[i] = (float)load_val(vals, dtype, i); }
}

// indptr[r] = first position whose row >= r (rows non-decreasing, strided int64)
__global__ void indptr_from_rows_kernel(const int64_t* __restrict__ rows, int64_t rs, int64_t nnz, int64_t n_rows,
                                        int64_t* __restrict__ indptr) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r > n_rows) return;
    int64_t lo = 0, hi = nnz;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (rows[mid * rs] < r) lo = mid + 1; else hi = mid;
    }
    indptr[r] = lo;
}

__global__ void coo_keys_kernel(const int64_t* __restrict__ rows, int64_t rs, const int64_t* __restrict__ cols, int64_t cs,
                                const void* __restrict__ vals, int dtype, int drop_zeros, int64_t nnz, int64_t n_cols,
                                unsigned long long* __restrict__ keys, uint32_t* __restrict__ pos) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < nnz; i += stride) {
        const bool drop = drop_zeros && load_val(vals, dtype, i) == 0.0;
        keys[i] = drop ? ~0ull : (unsigned long long)rows[i * rs] * (unsigned long long)n_cols + (unsigned long long)cols[i * cs];
        pos[i] = (uint32_t)i;
    }
}

// head[i] = 1 where a new (row, col) starts among the kept entries (sorted keys; dropped entries carry key ~0)
__global__ void coo_heads_kernel(const unsigned long long* __restrict__ keys, int64_t nnz, int64_t* __restrict__ head) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < nnz; i += stride) {
        const unsigned long long k = keys[i];
        head[i] = (k != ~0ull && (i == 0 || keys[i - 1] != k)) ? 1 : 0;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) head[nnz] = 0;
}

// every head sums its run of duplicates in sorted (= input, the sort is stable) order and writes the unique entry; a sum
// of zero is kept as a stored zero (coo_matrix(...).tocsr() keeps explicit zeros and duplicates that cancel)
__global__ void coo_compact_kernel(const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ perm,
                                   const int64_t* __restrict__ slot /* exclusive scan of head */, const void* __restrict__ vals,
                                   int dtype, int64_t nnz, int64_t n_cols, int32_t* __restrict__ indices,
                                   float* __restrict__ values, unsigned long long* __restrict__ ukeys,
                                   int64_t* __restrict__ run_ptr /* optional: run_ptr[o + 1] = end of entry o's run */) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < nnz; i += stride) {
        const unsigned long long k = keys[i];
        if (k == ~0ull || (i > 0 && keys[i - 1] == k)) continue;
        double s = load_val(vals, dtype, perm[i]);      // not 0.0 + ...: a lone -0.0 stays -0.0, as scipy stores it
        int64_t j = i + 1;
        for (; j < nnz && keys[j] == k; ++j) s += load_val(vals, dtype, perm[j]);
        const int64_t o = slot[i];
        indices[o] = (int32_t)(k % (unsigned long long)n_cols);
        values[o] = (float)s;
        ukeys[o] = k;
        if (run_ptr) run_ptr[o + 1] = j;
    }
}

__global__ void iota_i64_kernel(int64_t* __restrict__ x, int64_t count) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < count; i += stride) x[i] = i;
}

__global__ void widen_u32_kernel(const uint32_t* __restrict__ x, int64_t count, int64_t* __restrict__ y) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < count; i += stride) y[i] = (int64_t)x[i];
}

// values[o] = the sum of table[levels[perm[j]]] over the run j in [run_ptr[o], run_ptr[o+1]): the first term, then the
// others added in double in run order, rounded once to float -- the order and precision coo_compact_kernel sums float32
// values in, and on the sorted path (runs of one) the plain copy coo_convert_sorted_kernel makes.  flags[0] |= 1 for a
// level outside [0, n_levels) (its entry gets NaN).
__global__ void csr_values_from_table_kernel(const int64_t* __restrict__ run_ptr, const int64_t* __restrict__ perm,
                                             const int64_t* __restrict__ levels, const float* __restrict__ table,
                                             int64_t n_levels, int64_t n_unique, float* __restrict__ values,
                                             int* __restrict__ flags) {
    int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int f = 0;
    for (; o < n_unique; o += stride) {
        const int64_t a = run_ptr[o], b = run_ptr[o + 1];
        double s = 0.0;
        bool bad = false;
        for (int64_t j = a; j < b; ++j) {
            const int64_t lv = levels[perm[j]];
            if (lv < 0 || lv >= n_levels) { bad = true; break; }
            const double t = (double)table[lv];
            s = (j == a) ? t : s + t;                    // the first term as it is: a lone -0.0 stays -0.0
        }
        if (bad) f = 1;
        values[o] = bad ? __int_as_float(0x7fc00000) : (float)s;
    }
    if (f) atomicOr(flags, f);
}

__global__ void indptr_from_keys_kernel(const unsigned long long* __restrict__ ukeys, int64_t n_unique, int64_t n_rows,
                                        int64_t n_cols, int64_t* __restrict__ indptr) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r > n_rows) return;
    const unsigned long long key = (unsigned long long)r * (unsigned long long)n_cols;
    int64_t lo = 0, hi = n_unique;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (ukeys[mid] < key) lo = mid + 1; else hi = mid;
    }
    indptr[r] = lo;
}

__global__ void shift_i64_kernel(int64_t* __restrict__ x, int64_t count, int64_t delta) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < count; i += stride) x[i] += delta;
}

}  // namespace

extern "C" int pb200_shift_i64(pb200_ctx* ctx, int64_t* x, int64_t count, int64_t delta) {
    PB_ENTER(ctx);
    if (count <= 0 || delta == 0) return PB200_OK;
    const int blocks = (int)std::min<int64_t>(ceil_div64(count, 256), 8 * (int64_t)ctx->num_sms);
    shift_i64_kernel<<<blocks, 256, 0, ctx->stream>>>(x, count, delta);
    ctx->stats[0] += 1;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

// pb200_coo_to_csr, and with perm_out / run_ptr_out (both or neither) pb200_coo_to_csr_runs
static int coo_to_csr_impl(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                           const int64_t* rows, int64_t row_stride, const int64_t* cols, int64_t col_stride,
                           const void* vals, int val_dtype, int drop_zeros, int require_sorted_rows,
                           int64_t* indptr_out, int32_t* indices_out, float* values_out, int64_t* nnz_out_host,
                           int64_t* perm_out, int64_t* run_ptr_out) {
    PB_REQUIRE(ctx, n_rows >= 0 && n_cols > 0 && nnz >= 0, "coo_to_csr: bad shape");
    PB_REQUIRE(ctx, n_cols < (int64_t)2147483647, "coo_to_csr: column count must fit int32");
    PB_REQUIRE(ctx, nnz < (int64_t)4294967295ll, "coo_to_csr: nnz must be < 2^32");
    PB_REQUIRE(ctx, row_stride >= 1 && col_stride >= 1, "coo_to_csr: strides are in elements, >= 1");
    PB_REQUIRE(ctx, vals == nullptr || val_dtype == PB200_F32 || val_dtype == PB200_F64, "coo_to_csr: values must be f32 or f64");
    PB_REQUIRE(ctx, nnz_out_host != nullptr && indptr_out != nullptr, "coo_to_csr: outputs are required");
    PB_REQUIRE(ctx, (double)n_rows * (double)n_cols < 1.8e19, "coo_to_csr: n_rows * n_cols must fit 64 bits");
    if (nnz == 0) {
        PB_CUDA(ctx, cudaMemsetAsync(indptr_out, 0, sizeof(int64_t) * (size_t)(n_rows + 1), ctx->stream));
        if (run_ptr_out) PB_CUDA(ctx, cudaMemsetAsync(run_ptr_out, 0, sizeof(int64_t), ctx->stream));
        *nnz_out_host = 0;
        return PB200_OK;
    }
    Scratch sc(ctx);
    const int blocks = 8 * ctx->num_sms;
    int* flags = nullptr;
    PB_TRY(sc.alloc(&flags, 1));
    PB_CUDA(ctx, cudaMemsetAsync(flags, 0, sizeof(int), ctx->stream));
    coo_check_kernel<<<blocks, 256, 0, ctx->stream>>>(rows, row_stride, cols, col_stride, vals, val_dtype, drop_zeros, nnz,
                                                      n_rows, n_cols, flags);
    int h_flags = 0;
    PB_CUDA(ctx, cudaMemcpyAsync(&h_flags, flags, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    PB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->stats[0] += 1;
    PB_REQUIRE(ctx, !(h_flags & 2), "coo_to_csr: index out of range");
    // the reference asserts this for test data (models.py:246: "calculations assume testset is sorted by users")
    PB_REQUIRE(ctx, !(require_sorted_rows && (h_flags & 8)), "coo_to_csr: rows must be sorted (non-decreasing)");
    if (!(h_flags & (1 | 4))) {
        // strictly increasing (row, col), nothing to drop: conversion only
        coo_convert_sorted_kernel<<<blocks, 256, 0, ctx->stream>>>(cols, col_stride, vals, val_dtype, nnz, indices_out, values_out);
        indptr_from_rows_kernel<<<(unsigned)ceil_div64(n_rows + 1, 256), 256, 0, ctx->stream>>>(rows, row_stride, nnz, n_rows, indptr_out);
        ctx->stats[0] += 2;
        if (perm_out) {                               // every entry is its own run
            iota_i64_kernel<<<blocks, 256, 0, ctx->stream>>>(perm_out, nnz);
            iota_i64_kernel<<<blocks, 256, 0, ctx->stream>>>(run_ptr_out, nnz + 1);
            ctx->stats[0] += 2;
        }
        PB_CUDA(ctx, cudaGetLastError());
        *nnz_out_host = nnz;
        return PB200_OK;
    }
    unsigned long long *keys = nullptr, *keys_sorted = nullptr, *ukeys = nullptr;
    uint32_t *pos = nullptr, *perm = nullptr;
    int64_t *head = nullptr, *slot = nullptr;
    PB_TRY(sc.alloc(&keys, (size_t)nnz));
    PB_TRY(sc.alloc(&keys_sorted, (size_t)nnz));
    PB_TRY(sc.alloc(&ukeys, (size_t)nnz));
    PB_TRY(sc.alloc(&pos, (size_t)nnz));
    PB_TRY(sc.alloc(&perm, (size_t)nnz));
    PB_TRY(sc.alloc(&head, (size_t)nnz + 1));
    PB_TRY(sc.alloc(&slot, (size_t)nnz + 1));
    coo_keys_kernel<<<blocks, 256, 0, ctx->stream>>>(rows, row_stride, cols, col_stride, vals, val_dtype, drop_zeros, nnz, n_cols, keys, pos);
    int bits = 1;
    while (bits < 64 && ((double)n_rows * (double)n_cols) > std::ldexp(1.0, bits)) ++bits;
    if (h_flags & 4) bits = 64;                       // dropped entries carry the all-ones key and must sort last
    size_t temp_bytes = 0, scan_bytes = 0;
    PB_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, keys, keys_sorted, pos, perm, nnz, 0, bits, ctx->stream));
    PB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, head, slot, nnz + 1, ctx->stream));
    uint8_t* temp = nullptr;
    PB_TRY(sc.alloc(&temp, std::max(temp_bytes, scan_bytes)));
    PB_CUDA(ctx, cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys, keys_sorted, pos, perm, nnz, 0, bits, ctx->stream));
    coo_heads_kernel<<<blocks, 256, 0, ctx->stream>>>(keys_sorted, nnz, head);
    PB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(temp, scan_bytes, head, slot, nnz + 1, ctx->stream));
    coo_compact_kernel<<<blocks, 256, 0, ctx->stream>>>(keys_sorted, perm, slot, vals, val_dtype, nnz, n_cols, indices_out,
                                                        values_out, ukeys, run_ptr_out);
    if (perm_out) {
        PB_CUDA(ctx, cudaMemsetAsync(run_ptr_out, 0, sizeof(int64_t), ctx->stream));
        widen_u32_kernel<<<blocks, 256, 0, ctx->stream>>>(perm, nnz, perm_out);
        ctx->stats[0] += 1;
    }
    int64_t n_unique = 0;
    PB_CUDA(ctx, cudaMemcpyAsync(&n_unique, slot + nnz, sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->stream));
    PB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    indptr_from_keys_kernel<<<(unsigned)ceil_div64(n_rows + 1, 256), 256, 0, ctx->stream>>>(ukeys, n_unique, n_rows, n_cols, indptr_out);
    ctx->stats[0] += 6;
    PB_CUDA(ctx, cudaGetLastError());
    *nnz_out_host = n_unique;
    return PB200_OK;
}

extern "C" int pb200_coo_to_csr(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                                const int64_t* rows, int64_t row_stride, const int64_t* cols, int64_t col_stride,
                                const void* vals, int val_dtype, int drop_zeros, int require_sorted_rows,
                                int64_t* indptr_out, int32_t* indices_out, float* values_out, int64_t* nnz_out_host) {
    PB_ENTER(ctx);
    return coo_to_csr_impl(ctx, n_rows, n_cols, nnz, rows, row_stride, cols, col_stride, vals, val_dtype, drop_zeros,
                           require_sorted_rows, indptr_out, indices_out, values_out, nnz_out_host, nullptr, nullptr);
}

extern "C" int pb200_coo_to_csr_runs(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                                     const int64_t* rows, int64_t row_stride, const int64_t* cols, int64_t col_stride,
                                     const void* vals, int val_dtype, int drop_zeros, int require_sorted_rows,
                                     int64_t* indptr_out, int32_t* indices_out, float* values_out,
                                     int64_t* nnz_out_host, int64_t* perm_out, int64_t* run_ptr_out) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, run_ptr_out != nullptr && (perm_out != nullptr || nnz == 0), "coo_to_csr_runs: outputs are required");
    return coo_to_csr_impl(ctx, n_rows, n_cols, nnz, rows, row_stride, cols, col_stride, vals, val_dtype, drop_zeros,
                           require_sorted_rows, indptr_out, indices_out, values_out, nnz_out_host, perm_out, run_ptr_out);
}

extern "C" int pb200_csr_values_from_table(pb200_ctx* ctx, int64_t n_unique, const int64_t* run_ptr, const int64_t* perm,
                                           const int64_t* levels, const float* table, int64_t n_levels,
                                           float* values_out) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, n_unique >= 0 && n_levels >= 1, "csr_values_from_table: bad sizes");
    PB_REQUIRE(ctx, n_unique == 0 || (run_ptr && perm && levels && table && values_out),
               "csr_values_from_table: null pointer");
    if (n_unique == 0) return PB200_OK;
    Scratch sc(ctx);
    int* flags = nullptr;
    PB_TRY(sc.alloc(&flags, 1));
    PB_CUDA(ctx, cudaMemsetAsync(flags, 0, sizeof(int), ctx->stream));
    const int blocks = (int)std::min<int64_t>(ceil_div64(n_unique, 256), 8 * (int64_t)ctx->num_sms);
    csr_values_from_table_kernel<<<blocks, 256, 0, ctx->stream>>>(run_ptr, perm, levels, table, n_levels, n_unique,
                                                                  values_out, flags);
    ctx->stats[0] += 1;
    PB_CUDA(ctx, cudaGetLastError());
    int h_flags = 0;
    PB_CUDA(ctx, cudaMemcpyAsync(&h_flags, flags, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    PB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    PB_REQUIRE(ctx, !h_flags, "csr_values_from_table: a level is outside the table");
    return PB200_OK;
}

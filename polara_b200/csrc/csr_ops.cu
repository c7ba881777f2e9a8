// CSR format helpers: transpose (A -> CSR of A^T) and the ScaledSVD row/column scaling.
//
// The transpose is a one-time format conversion per build() (scipy does the analogous
// coo->csr/csc conversion at polara/recommender/models.py:169-174).  It is a stable
// radix sort of nnz positions keyed by column (CUB DeviceRadixSort -- library code, used
// for this format conversion only, not on the scoring hot path), followed by gathers.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace {

__global__ void expand_rows_kernel(const int64_t* __restrict__ indptr, int64_t n_rows, int32_t* __restrict__ rows,
                                   uint32_t* __restrict__ pos, int64_t nnz) {
    // one warp per row
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = w; r < n_rows; r += nw) {
        int64_t b = indptr[r], e = indptr[r + 1];
        for (int64_t p = b + lane; p < e; p += 32) { rows[p] = (int32_t)r; pos[p] = (uint32_t)p; }
    }
}

__global__ void gather_transposed_kernel(const uint32_t* __restrict__ perm, const int32_t* __restrict__ rows,
                                         const float* __restrict__ values, int64_t nnz,
                                         int32_t* __restrict__ t_indices, float* __restrict__ t_values) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < nnz; i += stride) {
        uint32_t p = perm[i];
        t_indices[i] = rows[p];
        t_values[i] = values[p];
    }
}

__global__ void gather_group_kernel(const uint32_t* __restrict__ perm, const int32_t* __restrict__ a,
                                    const int32_t* __restrict__ b, const float* __restrict__ val, int64_t nnz,
                                    int32_t* __restrict__ ao, int32_t* __restrict__ bo, float* __restrict__ vo) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < nnz; i += stride) {
        uint32_t p = perm[i];
        ao[i] = a[p]; bo[i] = b[p]; vo[i] = val[p];
    }
}

__global__ void iota_kernel(uint32_t* __restrict__ pos, int64_t nnz) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < nnz; i += stride) pos[i] = (uint32_t)i;
}

__global__ void indptr_from_sorted_kernel(const int32_t* __restrict__ sorted_keys, int64_t nnz, int64_t n_keys,
                                          int64_t* __restrict__ indptr) {
    int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c > n_keys) return;
    // first position whose key >= c
    int64_t lo = 0, hi = nnz;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if ((int64_t)sorted_keys[mid] < c) lo = mid + 1; else hi = mid;
    }
    indptr[c] = lo;
}

// nonzero values per column: stored zeros (explicit zero feedback, duplicates that cancel) are not counted
__global__ void count_cols_kernel(const int32_t* __restrict__ indices, const float* __restrict__ values, int64_t nnz,
                                  int32_t* __restrict__ counts) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < nnz; i += stride)
        if (values[i] != 0.0f) atomicAdd(counts + indices[i], 1);   // integer counts: order-independent
}

__global__ void rescale_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                               float* __restrict__ values, int64_t n_rows, const int32_t* __restrict__ col_counts,
                               double row_pow, double col_pow, int do_rows, int do_cols) {
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = w; r < n_rows; r += nw) {
        int64_t b = indptr[r], e = indptr[r + 1];
        // matrices.py:78-83: norm = sqrt(count); factor = norm**(scaling-1) where norm != 0
        double rf = 1.0;
        if (do_rows && e > b) rf = pow(sqrt((double)(e - b)), row_pow);
        for (int64_t p = b + lane; p < e; p += 32) {
            double v = (double)values[p] * rf;
            if (do_cols) {
                // a column without nonzeros keeps factor 1 (pow(0, <0) would be inf, and 0 * inf NaN): only stored zeros
                // meet it, and the reference has dropped them
                const int32_t cnt = col_counts[indices[p]];
                if (cnt > 0) v *= pow(sqrt((double)cnt), col_pow);
            }
            values[p] = (float)v;
        }
    }
}

// ---- panel-major copy (pb200_csr_block_columns) --------------------------------------------------------------------
// counts[p * n_rows + row] = nnz of `row` whose column lies in panel p; segstart = where that run begins in the source
__global__ void panel_count_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, int64_t n_rows,
                                   int64_t panel_cols, int n_panels, int64_t* __restrict__ counts,
                                   int64_t* __restrict__ segstart) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_rows * n_panels) return;
    const int64_t row = e % n_rows;
    const int p = (int)(e / n_rows);
    const int64_t beg = indptr[row], end = indptr[row + 1];
    auto first_ge = [&](int64_t colkey) {                 // columns are sorted inside a row
        int64_t lo = beg, hi = end;
        while (lo < hi) {
            int64_t mid = (lo + hi) >> 1;
            if ((int64_t)__ldg(indices + mid) < colkey) lo = mid + 1; else hi = mid;
        }
        return lo;
    };
    const int64_t a = first_ge((int64_t)p * panel_cols), b = first_ge((int64_t)(p + 1) * panel_cols);
    counts[e] = b - a;
    segstart[e] = a;
}

// one warp per (panel, row) run: copy it to its place in the panel-major arrays
__global__ void panel_scatter_kernel(const int64_t* __restrict__ b_indptr, const int64_t* __restrict__ segstart,
                                     const int32_t* __restrict__ indices, const float* __restrict__ values,
                                     int64_t n_vrows, int32_t* __restrict__ b_indices, float* __restrict__ b_values) {
    const int lane = threadIdx.x & 31;
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (; w < n_vrows; w += nw) {
        const int64_t dst = b_indptr[w], len = b_indptr[w + 1] - dst, src = segstart[w];
        for (int64_t t = lane; t < len; t += 32) { b_indices[dst + t] = indices[src + t]; b_values[dst + t] = values[src + t]; }
    }
}

}  // namespace

extern "C" int pb200_csr_block_columns(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                                       const int64_t* indptr, const int32_t* indices, const float* values,
                                       int64_t panel_cols, int n_panels, int64_t* b_indptr, int32_t* b_indices,
                                       float* b_values, int64_t* panel_ptr_host) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, panel_cols > 0 && n_panels >= 1 && n_panels <= 65536, "block_columns: bad panel shape");
    PB_REQUIRE(ctx, (int64_t)n_panels == std::max<int64_t>(1, ceil_div64(n_cols, panel_cols)),
               "block_columns: n_panels must be ceil(n_cols / panel_cols)");
    PB_REQUIRE(ctx, panel_ptr_host != nullptr, "block_columns: panel_ptr_host is required");
    const int64_t n_vrows = n_rows * n_panels;
    Scratch sc(ctx);
    int64_t *counts = nullptr, *segstart = nullptr;
    PB_TRY(sc.alloc(&counts, (size_t)n_vrows + 1));
    PB_TRY(sc.alloc(&segstart, (size_t)n_vrows + 1));
    PB_CUDA(ctx, cudaMemsetAsync(counts + n_vrows, 0, sizeof(int64_t), ctx->stream));
    if (n_vrows > 0)
        panel_count_kernel<<<(unsigned)ceil_div64(n_vrows, 256), 256, 0, ctx->stream>>>(indptr, indices, n_rows, panel_cols,
                                                                                       n_panels, counts, segstart);
    size_t temp_bytes = 0;
    PB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, temp_bytes, counts, b_indptr, n_vrows + 1, ctx->stream));
    uint8_t* temp = nullptr;
    PB_TRY(sc.alloc(&temp, temp_bytes));
    PB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(temp, temp_bytes, counts, b_indptr, n_vrows + 1, ctx->stream));
    if (n_vrows > 0 && nnz > 0)
        panel_scatter_kernel<<<8 * ctx->num_sms, 256, 0, ctx->stream>>>(b_indptr, segstart, indices, values, n_vrows,
                                                                        b_indices, b_values);
    ctx->stats[0] += 3;
    PB_CUDA(ctx, cudaGetLastError());
    // panel offsets back to the host (strided gather of n_panels + 1 pointers)
    PB_CUDA(ctx, cudaMemcpy2DAsync(panel_ptr_host, sizeof(int64_t), b_indptr, sizeof(int64_t) * (size_t)std::max<int64_t>(n_rows, 1),
                                   sizeof(int64_t), (size_t)(n_rows > 0 ? n_panels + 1 : 1), cudaMemcpyDeviceToHost, ctx->stream));
    PB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (n_rows == 0) for (int p = 0; p <= n_panels; ++p) panel_ptr_host[p] = 0;
    return PB200_OK;
}

extern "C" int pb200_csr_transpose(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                                   const int64_t* indptr, const int32_t* indices, const float* values,
                                   int64_t* t_indptr, int32_t* t_indices, float* t_values) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, nnz < (int64_t)4294967295ll, "transpose: nnz must be < 2^32");
    PB_REQUIRE(ctx, n_cols < (int64_t)2147483647 && n_rows < (int64_t)2147483647, "transpose: dimension must fit int32");
    Scratch sc(ctx);
    int32_t *rows = nullptr, *keys_out = nullptr;
    uint32_t *pos = nullptr, *perm = nullptr;
    PB_TRY(sc.alloc(&rows, (size_t)nnz));
    PB_TRY(sc.alloc(&keys_out, (size_t)nnz));
    PB_TRY(sc.alloc(&pos, (size_t)nnz));
    PB_TRY(sc.alloc(&perm, (size_t)nnz));
    int blocks = 8 * ctx->num_sms;
    expand_rows_kernel<<<blocks, 256, 0, ctx->stream>>>(indptr, n_rows, rows, pos, nnz);
    int bits = 1;
    while (((int64_t)1 << bits) < n_cols) ++bits;
    size_t temp_bytes = 0;
    PB_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, indices, keys_out, pos, perm, nnz, 0, bits, ctx->stream));
    uint8_t* temp = nullptr;
    PB_TRY(sc.alloc(&temp, temp_bytes));
    PB_CUDA(ctx, cub::DeviceRadixSort::SortPairs(temp, temp_bytes, indices, keys_out, pos, perm, nnz, 0, bits, ctx->stream));
    gather_transposed_kernel<<<blocks, 256, 0, ctx->stream>>>(perm, rows, values, nnz, t_indices, t_values);
    indptr_from_sorted_kernel<<<(unsigned)ceil_div64(n_cols + 1, 256), 256, 0, ctx->stream>>>(keys_out, nnz, n_cols, t_indptr);
    ctx->stats[0] += 4;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

extern "C" int pb200_rescale(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                             const int64_t* indptr, const int32_t* indices, float* values,
                             double row_scaling, double col_scaling) {
    PB_ENTER(ctx);
    int do_rows = row_scaling != 1.0, do_cols = col_scaling != 1.0;
    if (!do_rows && !do_cols) return PB200_OK;
    Scratch sc(ctx);
    int32_t* counts = nullptr;
    PB_TRY(sc.alloc(&counts, (size_t)n_cols));
    int blocks = 8 * ctx->num_sms;
    if (do_cols) {
        PB_CUDA(ctx, cudaMemsetAsync(counts, 0, sizeof(int32_t) * (size_t)n_cols, ctx->stream));
        count_cols_kernel<<<blocks, 256, 0, ctx->stream>>>(indices, values, nnz, counts);
        ctx->stats[0] += 1;
        PB_TRY(pb_reduce(ctx, counts, n_cols, PB200_I32));       // row-sharded matrix: column counts are global
    }
    // NOTE the reference scales rows first, then columns, each pass a sparse product with a diagonal matrix
    // (models.py:891-895, matrices.py:71-93, binary=True).  The row counts are structural: they include the stored zeros
    // of the ingested matrix.  The row pass is a sparse product even at row_scaling == 1, and a sparse product stores only
    // nonzero results, so the column counts see the matrix without its zeros: count_cols_kernel counts values != 0.
    // Scaling never turns a nonzero into a zero here, so both factors can be applied in one pass; zeros stay stored as 0.
    rescale_kernel<<<blocks, 256, 0, ctx->stream>>>(indptr, indices, values, n_rows, counts,
                                                    row_scaling - 1.0, col_scaling - 1.0, do_rows, do_cols);
    ctx->stats[0] += 1;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

// Stable grouping of a 3-way COO tensor by one mode (arrange_indices, polara/lib/sparse.py:239-264,
// does the analogous host-side preparation for dttm_par).
extern "C" int pb200_coo_group(pb200_ctx* ctx, int64_t nnz, int64_t n_keys, const int32_t* key, const int32_t* a,
                               const int32_t* b, const float* val, int64_t* seg_ptr, int32_t* a_out,
                               int32_t* b_out, float* val_out) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, nnz < (int64_t)4294967295ll && n_keys > 0, "coo_group: nnz must be < 2^32, n_keys > 0");
    Scratch sc(ctx);
    int32_t* keys_out = nullptr;
    uint32_t *pos = nullptr, *perm = nullptr;
    PB_TRY(sc.alloc(&keys_out, (size_t)nnz));
    PB_TRY(sc.alloc(&pos, (size_t)nnz));
    PB_TRY(sc.alloc(&perm, (size_t)nnz));
    int blocks = 8 * ctx->num_sms;
    iota_kernel<<<blocks, 256, 0, ctx->stream>>>(pos, nnz);
    int bits = 1;
    while (((int64_t)1 << bits) < n_keys) ++bits;
    size_t temp_bytes = 0;
    PB_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, key, keys_out, pos, perm, nnz, 0, bits, ctx->stream));
    uint8_t* temp = nullptr;
    PB_TRY(sc.alloc(&temp, temp_bytes));
    PB_CUDA(ctx, cub::DeviceRadixSort::SortPairs(temp, temp_bytes, key, keys_out, pos, perm, nnz, 0, bits, ctx->stream));
    gather_group_kernel<<<blocks, 256, 0, ctx->stream>>>(perm, a, b, val, nnz, a_out, b_out, val_out);
    indptr_from_sorted_kernel<<<(unsigned)ceil_div64(n_keys + 1, 256), 256, 0, ctx->stream>>>(keys_out, nnz, n_keys, seg_ptr);
    ctx->stats[0] += 4;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

// Factor rotation of the Tucker-rank sweep: V_r = fp32(V R) with V fp64 [n x K] and R fp64 [K x r] (the rotation that
// rounding one mode of the core gives its factor, CoffeeModel._check_reduced_rank, models.py:949-963), written as the
// zero-padded float32 operand the SpMM and scoring kernels read.
//
// Summation order (the contract the exact tests emulate): acc = 0.0, then acc = acc + V[i,k] * R[k,j] for k ascending,
// the product and the sum each rounded to fp64 (__dmul_rn / __dadd_rn: no FMA contraction), then one rounding to fp32.
// numpy's elementwise fp64 multiply and add reproduce every bit.
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int ROT_ROWS = 32;       // output rows per block (8 warps x 4 rows)
constexpr int ROT_COLS = 32;       // output columns per block (one per lane)
constexpr int ROT_KC = 32;         // K chunk staged in shared memory

// block (bx, by): rows [32 bx, 32 bx + 32) x columns [32 by, 32 by + 32) of the output; each K chunk stages its slice of
// the V rows and of R in shared memory, so every V element is read from memory once per column block
__global__ void __launch_bounds__(256) rotate_factor_kernel(int64_t n, int K, int r, const double* __restrict__ V,
                                                            int64_t ldv, const double* __restrict__ R, int64_t ldr,
                                                            float* __restrict__ out, int64_t ldo) {
    __shared__ double vs[ROT_ROWS][ROT_KC + 1];
    __shared__ double rs[ROT_KC][ROT_COLS];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int64_t row0 = (int64_t)blockIdx.x * ROT_ROWS;
    const int j = blockIdx.y * ROT_COLS + tx;
    double acc[ROT_ROWS / 8];
#pragma unroll
    for (int q = 0; q < ROT_ROWS / 8; ++q) acc[q] = 0.0;
    for (int k0 = 0; k0 < K; k0 += ROT_KC) {
        const int kc = min(ROT_KC, K - k0);
        for (int t = threadIdx.x; t < ROT_ROWS * ROT_KC; t += blockDim.x) {
            const int i = t / ROT_KC, k = t % ROT_KC;
            const int64_t row = row0 + i;
            vs[i][k] = (row < n && k < kc) ? V[row * ldv + k0 + k] : 0.0;
        }
        for (int t = threadIdx.x; t < ROT_KC * ROT_COLS; t += blockDim.x) {
            const int k = t / ROT_COLS, c = t % ROT_COLS;
            const int jj = blockIdx.y * ROT_COLS + c;
            rs[k][c] = (k < kc && jj < r) ? R[(int64_t)(k0 + k) * ldr + jj] : 0.0;
        }
        __syncthreads();
        for (int k = 0; k < kc; ++k) {
            const double b = rs[k][tx];
#pragma unroll
            for (int q = 0; q < ROT_ROWS / 8; ++q) acc[q] = __dadd_rn(acc[q], __dmul_rn(vs[ty + 8 * q][k], b));
        }
        __syncthreads();
    }
    if (j >= ldo) return;
#pragma unroll
    for (int q = 0; q < ROT_ROWS / 8; ++q) {
        const int64_t row = row0 + ty + 8 * q;
        if (row < n) out[row * ldo + j] = j < r ? __double2float_rn(acc[q]) : 0.0f;
    }
}

}  // namespace

extern "C" int pb200_rotate_factor(pb200_ctx* ctx, int64_t n, int K, int r, const double* V, int64_t ldv,
                                   const double* R, int64_t ldr, float* out, int64_t ldo) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, n >= 0 && K >= 1 && K <= 1024 && r >= 1 && r <= 1024, "rotate_factor: need 1 <= K, r <= 1024");
    PB_REQUIRE(ctx, ldv >= K && ldr >= r && ldo >= r, "rotate_factor: leading dimensions too small");
    PB_REQUIRE(ctx, ldo <= 65535LL * ROT_COLS, "rotate_factor: output leading dimension too large");
    if (n == 0) return PB200_OK;
    PB_REQUIRE(ctx, V && R && out, "rotate_factor: null pointer");
    const dim3 grid((unsigned)ceil_div64(n, ROT_ROWS), (unsigned)ceil_div64(ldo, ROT_COLS));
    rotate_factor_kernel<<<grid, 256, 0, ctx->stream>>>(n, K, r, V, ldv, R, ldr, out, ldo);
    ctx->stats[0] += 1;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

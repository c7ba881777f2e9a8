// Small dense building blocks of the randomized SVD / HOOI drivers:
//   gram (fp64 accumulation, deterministic two-stage reduction), one-sided Jacobi
//   eigensolver for symmetric PSD matrices (single CTA, fp64), tall x small GEMM,
//   counter-based Gaussian fill, SVQB orthonormalisation.
// These replace the LAPACK/ARPACK internals of scipy.sparse.linalg.svds
// (polara/recommender/models.py:844; polara/lib/tensor.py:71,75,79) and np.linalg.qr
// (polara/lib/tensor.py:61,63).
#include "common.cuh"

namespace {

// ------------------------------------------------------------------ gram ------
constexpr int GT = 64;        // G tile edge
constexpr int GR = 32;        // rows staged per step

__global__ void __launch_bounds__(256)
gram_partial_kernel(const float* __restrict__ Y, int64_t n, int c, int64_t ld, int64_t rows_per_block,
                    int tiles, double* __restrict__ partial /*[gridDim.x][tiles*(tiles+1)/2][GT*GT]*/) {
    // blockIdx.y enumerates upper-triangular tile pairs (ti <= tj)
    int ti = 0, tj = 0;
    {
        int t = blockIdx.y, row = 0;
        while (t >= tiles - row) { t -= tiles - row; ++row; }
        ti = row; tj = row + t;
    }
    __shared__ float sa[GR][GT + 4];
    __shared__ float sb[GR][GT + 4];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;   // 16 x 16 threads, 4x4 entries each
    double acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
    const int64_t r1 = min(n, r0 + rows_per_block);
    for (int64_t base = r0; base < r1; base += GR) {
        // cooperative load: GR x GT floats per operand = 2048 -> 8 per thread
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            int e = threadIdx.x + it * 256;
            int rr = e >> 6, cc = e & 63;
            int64_t row = base + rr;
            int ca = ti * GT + cc, cb = tj * GT + cc;
            float va = 0.f, vb = 0.f;
            if (row < r1) {
                if (ca < c) va = __ldg(Y + row * ld + ca);
                if (cb < c) vb = __ldg(Y + row * ld + cb);
            }
            sa[rr][cc] = va;
            sb[rr][cc] = vb;
        }
        __syncthreads();
#pragma unroll 4
        for (int rr = 0; rr < GR; ++rr) {
            float4 a4 = *reinterpret_cast<const float4*>(&sa[rr][ty * 4]);
            float4 b4 = *reinterpret_cast<const float4*>(&sb[rr][tx * 4]);
            double a[4] = {(double)a4.x, (double)a4.y, (double)a4.z, (double)a4.w};
            double b[4] = {(double)b4.x, (double)b4.y, (double)b4.z, (double)b4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    double* out = partial + ((int64_t)blockIdx.x * gridDim.y + blockIdx.y) * (GT * GT);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) out[(ty * 4 + i) * GT + tx * 4 + j] = acc[i][j];
}

__global__ void gram_reduce_kernel(const double* __restrict__ partial, int nblk, int npairs, int tiles,
                                   int c, double* __restrict__ G) {
    int pair = blockIdx.x;
    int ti = 0, tj = 0;
    {
        int t = pair, row = 0;
        while (t >= tiles - row) { t -= tiles - row; ++row; }
        ti = row; tj = row + t;
    }
    for (int e = threadIdx.x; e < GT * GT; e += blockDim.x) {
        double s = 0.0;
        for (int b = 0; b < nblk; ++b) s += partial[((int64_t)b * npairs + pair) * (GT * GT) + e];
        int i = ti * GT + e / GT, j = tj * GT + e % GT;
        if (i < c && j < c) {
            G[(int64_t)i * c + j] = s;
            G[(int64_t)j * c + i] = s;
        }
    }
}

// cross Gram C = A^T B of two tall panels (all tile pairs; same two-stage deterministic reduction)
__global__ void __launch_bounds__(256)
xgram_dense_partial_kernel(const float* __restrict__ A, int ca, int64_t lda, const float* __restrict__ B, int cb,
                           int64_t ldb, int64_t n, int64_t rows_per_block, int tiles_b, double* __restrict__ partial) {
    const int ti = blockIdx.y / tiles_b, tj = blockIdx.y % tiles_b;
    __shared__ float sa[GR][GT + 4];
    __shared__ float sb[GR][GT + 4];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    double acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_block;
    const int64_t r1 = min(n, r0 + rows_per_block);
    for (int64_t base = r0; base < r1; base += GR) {
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            int e = threadIdx.x + it * 256;
            int rr = e >> 6, cc = e & 63;
            int64_t row = base + rr;
            int xa = ti * GT + cc, xb = tj * GT + cc;
            float va = 0.f, vb = 0.f;
            if (row < r1) {
                if (xa < ca) va = __ldg(A + row * lda + xa);
                if (xb < cb) vb = __ldg(B + row * ldb + xb);
            }
            sa[rr][cc] = va;
            sb[rr][cc] = vb;
        }
        __syncthreads();
#pragma unroll 4
        for (int rr = 0; rr < GR; ++rr) {
            float4 a4 = *reinterpret_cast<const float4*>(&sa[rr][ty * 4]);
            float4 b4 = *reinterpret_cast<const float4*>(&sb[rr][tx * 4]);
            double a[4] = {(double)a4.x, (double)a4.y, (double)a4.z, (double)a4.w};
            double b[4] = {(double)b4.x, (double)b4.y, (double)b4.z, (double)b4.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    double* out = partial + ((int64_t)blockIdx.x * gridDim.y + blockIdx.y) * (GT * GT);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) out[(ty * 4 + i) * GT + tx * 4 + j] = acc[i][j];
}

__global__ void xgram_dense_reduce_kernel(const double* __restrict__ partial, int nblk, int ntiles, int tiles_b, int ca,
                                          int cb, double* __restrict__ C) {
    const int tile = blockIdx.x, ti = tile / tiles_b, tj = tile % tiles_b;
    for (int e = threadIdx.x; e < GT * GT; e += blockDim.x) {
        int x = ti * GT + e / GT, y = tj * GT + e % GT;
        if (x >= ca || y >= cb) continue;
        double s = 0.0;
        for (int b = 0; b < nblk; ++b) s += partial[((int64_t)b * ntiles + tile) * (GT * GT) + e];
        C[(int64_t)x * cb + y] = s;
    }
}

// ------------------------------------------------- one-sided Jacobi (PSD eig) --
// Rows of X (= G, symmetric) are rotated until mutually orthogonal; the accumulated
// rotations (rows of R) are the eigenvectors, row norms the eigenvalues.
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void __launch_bounds__(1024)
jacobi_psd_kernel(double* __restrict__ X, double* __restrict__ R, int c, double* __restrict__ lam_out,
                  double* __restrict__ vec_out, int max_sweeps) {
    __shared__ int s_rot;
    __shared__ int s_order[1024];
    __shared__ double s_norm[1024];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int e = threadIdx.x; e < c * c; e += blockDim.x) R[e] = (e / c == e % c) ? 1.0 : 0.0;
    __syncthreads();
    const int np = (c + 1) & ~1;          // padded to even
    const int rounds = np - 1;
    for (int sweep = 0; sweep < max_sweeps; ++sweep) {
        if (threadIdx.x == 0) s_rot = 0;
        __syncthreads();
        for (int rd = 0; rd < rounds; ++rd) {
            for (int k = warp; k < np / 2; k += nwarps) {
                int p, q;
                if (k == 0) { p = np - 1; q = rd % (np - 1); }
                else { p = (rd + k) % (np - 1); q = (rd - k + (np - 1)) % (np - 1); }
                if (p >= c || q >= c) continue;
                if (p > q) { int t = p; p = q; q = t; }
                double* xp = X + (int64_t)p * c; double* xq = X + (int64_t)q * c;
                double a = 0, b = 0, g = 0;
                for (int i = lane; i < c; i += 32) { double u = xp[i], v = xq[i]; a += u * u; b += v * v; g += u * v; }
                a = warp_sum(a); b = warp_sum(b); g = warp_sum(g);
                if (fabs(g) <= 1e-15 * sqrt(a * b) || g == 0.0) continue;
                double zeta = (b - a) / (2.0 * g);
                double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
                double* rp = R + (int64_t)p * c; double* rq = R + (int64_t)q * c;
                for (int i = lane; i < c; i += 32) {
                    double u = xp[i], v = xq[i];
                    xp[i] = cs * u - sn * v; xq[i] = sn * u + cs * v;
                    double ru = rp[i], rv = rq[i];
                    rp[i] = cs * ru - sn * rv; rq[i] = sn * ru + cs * rv;
                }
                if (lane == 0) s_rot = 1;
            }
            __syncthreads();
        }
        int any = s_rot;
        __syncthreads();
        if (!any) break;
    }
    // eigenvalues = row norms; sort descending (rank sort, c <= 1024)
    for (int p = warp; p < c; p += nwarps) {
        double a = 0;
        for (int i = lane; i < c; i += 32) { double u = X[(int64_t)p * c + i]; a += u * u; }
        a = warp_sum(a);
        if (lane == 0) s_norm[p] = sqrt(a);
    }
    __syncthreads();
    for (int p = threadIdx.x; p < c; p += blockDim.x) {
        int rank = 0;
        double mine = s_norm[p];
        for (int q = 0; q < c; ++q) { double o = s_norm[q]; rank += (o > mine) || (o == mine && q < p); }
        s_order[rank] = p;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < c * c; e += blockDim.x) {
        int i = e / c, j = e % c;
        vec_out[e] = R[(int64_t)s_order[i] * c + j];
    }
    for (int p = threadIdx.x; p < c; p += blockDim.x) lam_out[p] = s_norm[s_order[p]];
}

// ---- the same one-sided Jacobi spread over the whole GPU: one launch per ROUND of a sweep (the c/2 row pairs of a round
// are disjoint), one block per pair.  The single-CTA kernel above does all c (c - 1) / 2 rotations of a sweep in one SM,
// which does not scale to c in the hundreds (a HOOI unfolding / the rank-500 build of C5).  Same pair order => same rotations.
__global__ void jacobi_init_kernel(double* __restrict__ R, int c, int* __restrict__ flags) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < c * c) R[e] = (e / c == e % c) ? 1.0 : 0.0;
    if (e < 64) flags[e] = 0;
}

__global__ void __launch_bounds__(128)
jacobi_round_kernel(double* __restrict__ X, double* __restrict__ R, int c, int np, int rd, int sweep,
                    int* __restrict__ flags /* flags[s] = rotations done in sweep s */) {
    // sweeps after the first one that rotated nothing are no-ops (the host enqueues a fixed number of sweeps)
    if (sweep > 0 && flags[sweep - 1] == 0) return;
    const int k = blockIdx.x;
    int p, q;
    if (k == 0) { p = np - 1; q = rd % (np - 1); }
    else { p = (rd + k) % (np - 1); q = (rd - k + (np - 1)) % (np - 1); }
    if (p >= c || q >= c) return;
    if (p > q) { int t = p; p = q; q = t; }
    double* xp = X + (int64_t)p * c; double* xq = X + (int64_t)q * c;
    double a = 0, b = 0, g = 0;
    for (int i = threadIdx.x; i < c; i += 128) { const double u = xp[i], v = xq[i]; a += u * u; b += v * v; g += u * v; }
    __shared__ double red[3][4];
    a = warp_sum(a); b = warp_sum(b); g = warp_sum(g);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { red[0][warp] = a; red[1][warp] = b; red[2][warp] = g; }
    __syncthreads();
    a = red[0][0] + red[0][1] + red[0][2] + red[0][3];
    b = red[1][0] + red[1][1] + red[1][2] + red[1][3];
    g = red[2][0] + red[2][1] + red[2][2] + red[2][3];
    if (fabs(g) <= 1e-15 * sqrt(a * b) || g == 0.0) return;
    const double zeta = (b - a) / (2.0 * g);
    const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
    const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
    double* rp = R + (int64_t)p * c; double* rq = R + (int64_t)q * c;
    for (int i = threadIdx.x; i < c; i += 128) {
        const double u = xp[i], v = xq[i];
        xp[i] = cs * u - sn * v; xq[i] = sn * u + cs * v;
        const double ru = rp[i], rv = rq[i];
        rp[i] = cs * ru - sn * rv; rq[i] = sn * ru + cs * rv;
    }
    if (threadIdx.x == 0) flags[sweep] = 1;
}

// eigenvalues = row norms of the rotated X, sorted descending; eigenvectors = the matching rows of R
__global__ void __launch_bounds__(1024)
jacobi_finish_kernel(const double* __restrict__ X, const double* __restrict__ R, int c, double* __restrict__ lam_out,
                     double* __restrict__ vec_out) {
    __shared__ int s_order[1024];
    __shared__ double s_norm[1024];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int p = warp; p < c; p += nwarps) {
        double a = 0;
        for (int i = lane; i < c; i += 32) { const double u = X[(int64_t)p * c + i]; a += u * u; }
        a = warp_sum(a);
        if (lane == 0) s_norm[p] = sqrt(a);
    }
    __syncthreads();
    for (int p = threadIdx.x; p < c; p += blockDim.x) {
        int rank = 0;
        const double mine = s_norm[p];
        for (int q = 0; q < c; ++q) { const double o = s_norm[q]; rank += (o > mine) || (o == mine && q < p); }
        s_order[rank] = p;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < c * c; e += blockDim.x) vec_out[e] = R[(int64_t)s_order[e / c] * c + e % c];
    for (int p = threadIdx.x; p < c; p += blockDim.x) lam_out[p] = s_norm[s_order[p]];
}

// ------------------------------------------------------- tall x small GEMM ----
constexpr int RM_BM = 128, RM_BN = 64, RM_BK = 16;
__global__ void __launch_bounds__(256)
right_multiply_kernel(const float* __restrict__ Y, int64_t n, int c, int64_t ldy,
                      const float* __restrict__ W, int c2, int64_t ldw, float* __restrict__ C, int64_t ldc) {
    __shared__ float sy[RM_BK][RM_BM + 4];
    __shared__ float sw[RM_BK][RM_BN + 4];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;     // 16 x 16, micro tile 8 rows x 4 cols
    const int64_t row0 = (int64_t)blockIdx.x * RM_BM;
    const int col0 = blockIdx.y * RM_BN;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < c; k0 += RM_BK) {
        // Y tile: 128 rows x 16 k = 2048 -> 8 per thread ; coalesced along k
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            int e = threadIdx.x + it * 256;
            int rr = e >> 4, kk = e & 15;
            int64_t row = row0 + rr;
            float v = 0.f;
            if (row < n && k0 + kk < c) v = __ldg(Y + row * ldy + k0 + kk);
            sy[kk][rr] = v;
        }
        // W tile: 16 k x 64 cols = 1024 -> 4 per thread
#pragma unroll
        for (int it = 0; it < 4; ++it) {
            int e = threadIdx.x + it * 256;
            int kk = e >> 6, cc = e & 63;
            float v = 0.f;
            if (k0 + kk < c && col0 + cc < c2) v = __ldg(W + (int64_t)(k0 + kk) * ldw + col0 + cc);
            sw[kk][cc] = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < RM_BK; ++kk) {
            float4 y0 = *reinterpret_cast<const float4*>(&sy[kk][ty * 8]);
            float4 y1 = *reinterpret_cast<const float4*>(&sy[kk][ty * 8 + 4]);
            float4 w4 = *reinterpret_cast<const float4*>(&sw[kk][tx * 4]);
            float a[8] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w};
            float b[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        int64_t row = row0 + ty * 8 + i;
        if (row >= n) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int col = col0 + tx * 4 + j;
            if (col < c2) C[row * ldc + col] = acc[i][j];
        }
    }
}

// ------------------------------------------------------------ gaussian fill ---
__device__ __forceinline__ uint64_t mix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__global__ void gaussian_kernel(float* __restrict__ X, int64_t count, uint64_t seed) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t p = i; 2 * p < count; p += stride) {
        uint64_t h = mix64(seed * 0xD1342543DE82EF95ull + (uint64_t)p);
        uint32_t a = (uint32_t)(h >> 32), b = (uint32_t)h;
        float u1 = ((float)(a >> 8) + 0.5f) * (1.0f / 16777216.0f);
        float u2 = ((float)(b >> 8) + 0.5f) * (1.0f / 16777216.0f);
        float rad = sqrtf(-2.0f * logf(u1));
        float sn, cs;
        sincospif(2.0f * u2, &sn, &cs);
        X[2 * p] = rad * cs;
        if (2 * p + 1 < count) X[2 * p + 1] = rad * sn;
    }
}

// W[i][j] = vecs[j][i] * (lam[j] > cut ? lam[j]^-1/2 : 0)   (c x c, float32)
__global__ void svqb_matrix_kernel(const double* __restrict__ vecs, const double* __restrict__ lam, int c,
                                   float* __restrict__ W) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= c * c) return;
    int i = e / c, j = e % c;
    double l = lam[j], cut = lam[0] * 1e-12;
    double s = (l > cut && l > 0.0) ? rsqrt(l) : 0.0;
    W[e] = (float)(vecs[(int64_t)j * c + i] * s);
}

}  // namespace

int pb_gram(pb200_ctx* ctx, const float* Y, int64_t n, int c, int64_t ld, double* G) {
    PB_REQUIRE(ctx, c > 0 && c <= 1024, "gram: width must be in 1..1024");
    Scratch sc(ctx);
    int tiles = (c + GT - 1) / GT;
    int npairs = tiles * (tiles + 1) / 2;
    int nblk = (int)std::min<int64_t>(std::max<int64_t>(1, ceil_div64(n, 2048)), 2 * (int64_t)ctx->num_sms);
    int64_t rows_per_block = ceil_div64(std::max<int64_t>(n, 1), nblk);
    rows_per_block = ceil_div64(rows_per_block, GR) * GR;
    nblk = (int)std::max<int64_t>(1, ceil_div64(std::max<int64_t>(n, 1), rows_per_block));
    double* partial = nullptr;
    PB_TRY(sc.alloc(&partial, (size_t)nblk * npairs * GT * GT));
    gram_partial_kernel<<<dim3(nblk, npairs), 256, 0, ctx->stream>>>(Y, n, c, ld, rows_per_block, tiles, partial);
    gram_reduce_kernel<<<npairs, 256, 0, ctx->stream>>>(partial, nblk, npairs, tiles, c, G);
    ctx->stats[0] += 2;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

int pb_cross_gram(pb200_ctx* ctx, const float* A, int ca, int64_t lda, const float* B, int cb, int64_t ldb, int64_t n,
                  double* C) {
    PB_REQUIRE(ctx, ca > 0 && cb > 0 && ca <= 1024 && cb <= 1024, "cross_gram: widths must be in 1..1024");
    Scratch sc(ctx);
    const int tiles_a = (ca + GT - 1) / GT, tiles_b = (cb + GT - 1) / GT, ntiles = tiles_a * tiles_b;
    int nblk = (int)std::min<int64_t>(std::max<int64_t>(1, ceil_div64(n, 2048)), 2 * (int64_t)ctx->num_sms);
    int64_t rows_per_block = ceil_div64(std::max<int64_t>(n, 1), nblk);
    rows_per_block = ceil_div64(rows_per_block, GR) * GR;
    nblk = (int)std::max<int64_t>(1, ceil_div64(std::max<int64_t>(n, 1), rows_per_block));
    double* partial = nullptr;
    PB_TRY(sc.alloc(&partial, (size_t)nblk * ntiles * GT * GT));
    xgram_dense_partial_kernel<<<dim3(nblk, ntiles), 256, 0, ctx->stream>>>(A, ca, lda, B, cb, ldb, n, rows_per_block,
                                                                            tiles_b, partial);
    xgram_dense_reduce_kernel<<<ntiles, 256, 0, ctx->stream>>>(partial, nblk, ntiles, tiles_b, ca, cb, C);
    ctx->stats[0] += 2;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

int pb_eig_psd(pb200_ctx* ctx, double* G, int c, double* lam, double* vecs) {
    PB_REQUIRE(ctx, c > 0 && c <= 1024, "eig: size must be in 1..1024");
    Scratch sc(ctx);
    double* R = nullptr;
    PB_TRY(sc.alloc(&R, (size_t)c * c));
    if (c >= 160) {
        // one launch per round, one block per row pair; a fixed budget of sweeps is enqueued and the rounds of a sweep turn
        // into no-ops once the sweep before rotated nothing (no host round trip)
        const int np = (c + 1) & ~1, rounds = np - 1, max_sweeps = 40, batch = 2;
        int* flags = nullptr;
        PB_TRY(sc.alloc(&flags, 64));
        jacobi_init_kernel<<<(c * c + 255) / 256, 256, 0, ctx->stream>>>(R, c, flags);
        int sweeps_done = 0;
        for (int s0 = 0; s0 < max_sweeps; s0 += batch) {
            for (int sweep = s0; sweep < s0 + batch; ++sweep)
                for (int rd = 0; rd < rounds; ++rd)
                    jacobi_round_kernel<<<np / 2, 128, 0, ctx->stream>>>(G, R, c, np, rd, sweep, flags);
            sweeps_done = s0 + batch;
            int h[2] = {1, 1};                              // did the two sweeps of this batch still rotate anything?
            PB_CUDA(ctx, cudaMemcpyAsync(h, flags + s0, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
            PB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            if (h[0] == 0 || h[1] == 0) break;
        }
        ctx->stats[0] += (uint64_t)sweeps_done * rounds;
        jacobi_finish_kernel<<<1, 1024, 0, ctx->stream>>>(G, R, c, lam, vecs);
        ctx->stats[0] += 2;
        PB_CUDA(ctx, cudaGetLastError());
        return PB200_OK;
    }
    jacobi_psd_kernel<<<1, 1024, 0, ctx->stream>>>(G, R, c, lam, vecs, 40);
    ctx->stats[0] += 1;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

int pb_right_multiply(pb200_ctx* ctx, const float* Y, int64_t n, int c, int64_t ldy, const float* W,
                      int c2, int64_t ldw, float* C, int64_t ldc) {
    if (n == 0 || c2 == 0) return PB200_OK;
    dim3 grid((unsigned)ceil_div64(n, RM_BM), (unsigned)((c2 + RM_BN - 1) / RM_BN));
    right_multiply_kernel<<<grid, 256, 0, ctx->stream>>>(Y, n, c, ldy, W, c2, ldw, C, ldc);
    ctx->stats[0] += 1;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

int pb_fill_gaussian(pb200_ctx* ctx, float* X, int64_t count, uint64_t seed) {
    int blocks = (int)std::min<int64_t>(ceil_div64(std::max<int64_t>(count / 2, 1), 256), 8 * (int64_t)ctx->num_sms);
    gaussian_kernel<<<blocks, 256, 0, ctx->stream>>>(X, count, seed);
    ctx->stats[0] += 1;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

int pb_orthonormalize(pb200_ctx* ctx, const float* Y, int64_t n, int c, int64_t ldy, float* Q, int64_t ldq,
                      double* lam_out, bool rows_sharded) {
    Scratch sc(ctx);
    double *G = nullptr, *lam = nullptr, *vecs = nullptr;
    float* W = nullptr;
    PB_TRY(sc.alloc(&G, (size_t)c * c));
    PB_TRY(sc.alloc(&vecs, (size_t)c * c));
    PB_TRY(sc.alloc(&W, (size_t)c * c));
    if (lam_out) lam = lam_out; else PB_TRY(sc.alloc(&lam, (size_t)c));
    PB_TRY(pb_gram(ctx, Y, n, c, ldy, G));
    if (rows_sharded) PB_TRY(pb_reduce(ctx, G, (int64_t)c * c, PB200_F64));
    PB_TRY(pb_eig_psd(ctx, G, c, lam, vecs));
    svqb_matrix_kernel<<<(c * c + 255) / 256, 256, 0, ctx->stream>>>(vecs, lam, c, W);
    ctx->stats[0] += 1;
    PB_TRY(pb_right_multiply(ctx, Y, n, c, ldy, W, c, c, Q, ldq));
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

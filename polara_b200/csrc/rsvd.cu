// Truncated SVD by randomized subspace iteration (Halko/Martinsson/Tropp) on the sparse
// CSR matrix, and thin SVD of dense tall-skinny matrices.  Replaces
// scipy.sparse.linalg.svds (ARPACK) at polara/recommender/models.py:844 and at
// polara/lib/tensor.py:71,75,79.
//
//   Omega [n_cols x ell] ~ N(0,1)
//   W = orth(A Omega);  Q = orth(A^T W)
//   repeat: W = orth(A Q); Q = orth(A^T W)   until the leading Ritz values settle
//   B = A Q ; eig(B^T B) = Z L Z^T ; sigma = sqrt(L) ; V = Q Z ; U = B Z / sigma
//
// Row-sharded build (SURVEY.md 8e): with a reduce hook installed every rank passes ITS row block A_g (and A_g^T);
// the Gram matrices of the tall panels and the panel A^T W = sum_g A_g^T W_g are summed over the shards, everything
// on the item side (Omega, Q, eig, V, sigma) is computed redundantly and identically on every rank; U_out holds the
// rank's own rows.
//
// Factored operator (HybridSVD, pb200_rsvd_factored): A above stands for M = K_u^T A K_i, each product with M or M^T a
// chain of up to three SpMMs through two extra panels; the iteration itself is unchanged.
//
// All SpMMs are fp32 (spmm.cu); Gram matrices and the small eigenproblems are fp64.
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace {

// Singular values at or below 1e-6 * sigma_1 (Gram eigenvalues at or below 1e-12 * lam_1, the cut of svqb_matrix_kernel
// in dense.cu) are treated as zero: sigma_j = 0 and the left singular vector U = M v_j / sigma_j is a zero column instead
// of rounding noise amplified by 1 / sigma_j (DESIGN.md §4).
__device__ __forceinline__ bool live_sigma(const double* __restrict__ lam, int j) {
    const double l = lam[j];
    return l > 0.0 && l > 1e-12 * lam[0];
}

__global__ void take_columns_kernel(const double* __restrict__ vecs /*[c x c] rows=eigvecs*/, int c, int r,
                                    const double* __restrict__ lam, int scale_inv_sigma, float* __restrict__ W /*[c x r]*/) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= c * r) return;
    int i = e / r, j = e % r;
    double s = 1.0;
    if (scale_inv_sigma) s = live_sigma(lam, j) ? rsqrt(lam[j]) : 0.0;
    W[e] = (float)(vecs[(int64_t)j * c + i] * s);
}

__global__ void sqrt_leading_kernel(const double* __restrict__ lam, int r, double* __restrict__ sigma) {
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < r) sigma[j] = live_sigma(lam, j) ? sqrt(lam[j]) : 0.0;
}

__global__ void rows_to_float_kernel(const double* __restrict__ vecs, int c, int r, float* __restrict__ out) {
    int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < c * r) out[e] = (float)vecs[e];      // first r rows of vecs (row-major [c x c]) -> [r x c]
}

}  // namespace

// One product of the operator chain  Y = Last (Mid (First X))  with First / Last optional (NULL = identity): the
// subspace iteration of the factored operator M = K_u^T A K_i applies  M X = K_u^T (A (K_i X))  and
// M^T W = K_i^T (A^T (K_u W)).  tmp_first holds First X (rows of Mid's column space), tmp_mid holds Mid (...) when Last
// follows.  Every product is one SpMM (pb_spmm_view), so an identity factor (one unit nnz per row) copies exactly.
static int apply_chain(pb200_ctx* ctx, const pb200_csr_view* first, const pb200_csr_view* mid, const pb200_csr_view* last,
                       const float* X, float* tmp_first, float* tmp_mid, float* Y, int ell) {
    if (first) {
        PB_TRY(pb_spmm_view(ctx, first, X, ell, tmp_first, ell, ell));
        X = tmp_first;
    }
    if (!last) return pb_spmm_view(ctx, mid, X, ell, Y, ell, ell);
    PB_TRY(pb_spmm_view(ctx, mid, X, ell, tmp_mid, ell, ell));
    return pb_spmm_view(ctx, last, tmp_mid, ell, Y, ell, ell);
}

extern "C" int pb200_rsvd_factored(pb200_ctx* ctx, const pb200_csr_view* A, const pb200_csr_view* At,
                                   const pb200_csr_view* Ki, const pb200_csr_view* Kit,
                                   const pb200_csr_view* Ku, const pb200_csr_view* Kut,
                                   int rank, int ell, int max_iters, double tol, double vec_tol, uint64_t seed,
                                   float* V_out, int64_t ldv, double* sigma_out, float* U_out, int64_t ldu,
                                   double* info_host) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, A && At && A->indptr && At->indptr, "rsvd: null matrix view");
    const int64_t n_rows = A->n_rows, n_cols = A->n_cols;
    PB_REQUIRE(ctx, At->n_rows == n_cols && At->n_cols == n_rows && At->nnz == A->nnz, "rsvd: A^T does not match A");
    PB_REQUIRE(ctx, !Ki == !Kit && !Ku == !Kut, "rsvd: a factor needs both K and K^T (or neither)");
    PB_REQUIRE(ctx, !Ki || (Ki->indptr && Kit->indptr && Ki->n_rows == n_cols && Ki->n_cols == n_cols &&
                            Kit->n_rows == n_cols && Kit->n_cols == n_cols && Kit->nnz == Ki->nnz),
               "rsvd: the item factor K_i and K_i^T must be n_cols x n_cols (n_cols of A) with equal nnz");
    PB_REQUIRE(ctx, !Ku || (Ku->indptr && Kut->indptr && Ku->n_rows == n_rows && Ku->n_cols == n_rows &&
                            Kut->n_rows == n_rows && Kut->n_cols == n_rows && Kut->nnz == Ku->nnz),
               "rsvd: the user factor K_u and K_u^T must be n_rows x n_rows (n_rows of A) with equal nnz");
    if ((Ki || Ku) && ctx->reduce_fn) {
        ctx->err = "rsvd: factored operator under a reduce hook (row-sharded build) is not implemented: a user factor "
                   "mixes the rows of all shards";
        return PB200_ENOTIMPL;
    }
    PB_REQUIRE(ctx, rank > 0 && ell % 32 == 0 && ell >= rank && ell <= 1024, "rsvd: need 0 < rank <= ell <= 1024, ell % 32 == 0");
    PB_REQUIRE(ctx, rank <= n_cols && (rank <= n_rows || ctx->reduce_fn), "rsvd: rank exceeds matrix dimension");
    PB_REQUIRE(ctx, ldv >= rank && (!U_out || ldu >= rank), "rsvd: leading dimension smaller than rank");
    Scratch sc(ctx);
    float *Yn = nullptr, *Qn = nullptr, *Qprev = nullptr, *Ym = nullptr, *Wm = nullptr, *Wsmall = nullptr;
    float *Pi = nullptr, *Pu = nullptr;      // chain intermediates: item-side [n_cols x ell], user-side [n_rows x ell]
    double *lam = nullptr, *G = nullptr, *vecs = nullptr, *Cx = nullptr;
    PB_TRY(sc.alloc(&Yn, (size_t)n_cols * ell));
    PB_TRY(sc.alloc(&Qn, (size_t)n_cols * ell));
    PB_TRY(sc.alloc(&Qprev, (size_t)n_cols * ell));
    PB_TRY(sc.alloc(&Ym, (size_t)n_rows * ell));
    PB_TRY(sc.alloc(&Wm, (size_t)n_rows * ell));
    PB_TRY(sc.alloc(&Wsmall, (size_t)ell * ell));
    PB_TRY(sc.alloc(&lam, (size_t)ell));
    PB_TRY(sc.alloc(&G, (size_t)ell * ell));
    PB_TRY(sc.alloc(&vecs, (size_t)ell * ell));
    PB_TRY(sc.alloc(&Cx, (size_t)rank * rank));
    if (Ki || Ku) {
        PB_TRY(sc.alloc(&Pi, (size_t)n_cols * ell));
        PB_TRY(sc.alloc(&Pu, (size_t)n_rows * ell));
    }
    std::vector<double> prev(rank, 0.0), cur(ell, 0.0), cross((size_t)rank * rank, 0.0);

    PB_TRY(pb_fill_gaussian(ctx, Qn, n_cols * (int64_t)ell, seed));
    int iters = 0;
    double worst = 1.0, angle = 1.0;
    bool converged = false;
    for (int it = 0; it <= max_iters; ++it) {
        PB_TRY(apply_chain(ctx, Ki, A, Kut, Qn, Pi, Pu, Ym, ell));                     // M Q
        PB_TRY(pb_orthonormalize(ctx, Ym, n_rows, ell, ell, Wm, ell, nullptr, /*rows_sharded=*/true));
        PB_TRY(apply_chain(ctx, Ku, At, Kit, Wm, Pu, Pi, Yn, ell));                    // M^T W
        PB_TRY(pb_reduce(ctx, Yn, n_cols * (int64_t)ell, PB200_F32));     // A^T W = sum over row shards of A_g^T W_g
        std::swap(Qn, Qprev);
        PB_TRY(pb_orthonormalize(ctx, Yn, n_cols, ell, ell, Qn, ell, lam));
        iters = it;
        // (a) lam = eig(Yn^T Yn), Yn = A^T W with W orthonormal  ->  sqrt(lam) approximates sigma;
        // (b) the columns of Q are the Ritz vectors in that order: C = Qprev[:, :r]^T Q[:, :r] has the cosines of the
        //     principal angles between the leading-r subspaces of two successive iterates as singular values, so
        //     r - ||C||_F^2 = sum sin^2(theta_i) >= sin^2(theta_max)
        if (it > 0 && vec_tol > 0.0) PB_TRY(pb_cross_gram(ctx, Qprev, rank, ell, Qn, rank, ell, n_cols, Cx));
        PB_CUDA(ctx, cudaMemcpyAsync(cur.data(), lam, sizeof(double) * ell, cudaMemcpyDeviceToHost, ctx->stream));
        if (it > 0 && vec_tol > 0.0)
            PB_CUDA(ctx, cudaMemcpyAsync(cross.data(), Cx, sizeof(double) * (size_t)rank * rank, cudaMemcpyDeviceToHost, ctx->stream));
        PB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        worst = 0.0;
        for (int j = 0; j < rank; ++j) {
            double s = std::sqrt(std::max(cur[j], 0.0));
            double d = std::fabs(s - prev[j]) / std::max(s, 1e-300);
            worst = std::max(worst, d);
            prev[j] = s;
        }
        if (it > 0 && vec_tol > 0.0) {
            double fro = 0.0;
            for (double c : cross) fro += c * c;
            angle = std::sqrt(std::max(0.0, (double)rank - fro));
        } else if (vec_tol <= 0.0) {
            angle = 0.0;
        }
        if (it > 0 && worst < tol && angle <= std::max(vec_tol, 0.0)) { converged = true; break; }
    }
    // Rayleigh-Ritz on the final subspace: B = M Q (U = B Z / sigma are the left vectors of M)
    PB_TRY(apply_chain(ctx, Ki, A, Kut, Qn, Pi, Pu, Ym, ell));
    PB_TRY(pb_gram(ctx, Ym, n_rows, ell, ell, G));
    PB_TRY(pb_reduce(ctx, G, (int64_t)ell * ell, PB200_F64));
    PB_TRY(pb_eig_psd(ctx, G, ell, lam, vecs));
    sqrt_leading_kernel<<<(rank + 127) / 128, 128, 0, ctx->stream>>>(lam, rank, sigma_out);
    take_columns_kernel<<<(ell * rank + 255) / 256, 256, 0, ctx->stream>>>(vecs, ell, rank, lam, 0, Wsmall);
    PB_TRY(pb_right_multiply(ctx, Qn, n_cols, ell, ell, Wsmall, rank, rank, V_out, ldv));
    if (U_out) {
        take_columns_kernel<<<(ell * rank + 255) / 256, 256, 0, ctx->stream>>>(vecs, ell, rank, lam, 1, Wsmall);
        PB_TRY(pb_right_multiply(ctx, Ym, n_rows, ell, ell, Wsmall, rank, rank, U_out, ldu));
    }
    ctx->stats[0] += 3;
    PB_CUDA(ctx, cudaGetLastError());
    PB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (info_host) {
        info_host[0] = (double)iters; info_host[1] = worst; info_host[2] = angle; info_host[3] = converged ? 1.0 : 0.0;
        for (int i = 4; i < 8; ++i) info_host[i] = 0.0;
    }
    return PB200_OK;
}

extern "C" int pb200_rsvd_csr(pb200_ctx* ctx, const pb200_csr_view* A, const pb200_csr_view* At,
                              int rank, int ell, int max_iters, double tol, double vec_tol, uint64_t seed,
                              float* V_out, int64_t ldv, double* sigma_out, float* U_out, int64_t ldu,
                              double* info_host) {
    return pb200_rsvd_factored(ctx, A, At, nullptr, nullptr, nullptr, nullptr, rank, ell, max_iters, tol, vec_tol, seed,
                               V_out, ldv, sigma_out, U_out, ldu, info_host);
}

extern "C" int pb200_rsvd(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                          const int64_t* indptr, const int32_t* indices, const float* values,
                          const int64_t* t_indptr, const int32_t* t_indices, const float* t_values,
                          int rank, int ell, int max_iters, double tol, uint64_t seed,
                          float* V_out, int64_t ldv, double* sigma_out, float* U_out, int64_t ldu,
                          int* iters_done_host) {
    PB_ENTER(ctx);
    pb200_csr_view a{n_rows, n_cols, nnz, indptr, indices, values, 1, n_cols, nullptr};
    pb200_csr_view at{n_cols, n_rows, nnz, t_indptr, t_indices, t_values, 1, n_rows, nullptr};
    double info[8];
    int st = pb200_rsvd_csr(ctx, &a, &at, rank, ell, max_iters, tol, /*vec_tol=*/0.0, seed, V_out, ldv, sigma_out, U_out, ldu, info);
    if (st == PB200_OK && iters_done_host) *iters_done_host = (int)info[0];
    return st;
}

extern "C" int pb200_tall_svd(pb200_ctx* ctx, const float* M, int64_t n, int c, int64_t ldm, int rank,
                              double* sigma_out, float* U_out, int64_t ldu, float* Vt_out) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, c > 0 && c <= 1024 && rank > 0 && rank <= c, "tall_svd: need 0 < rank <= c <= 1024");
    PB_REQUIRE(ctx, ldm >= c && ldu >= rank, "tall_svd: leading dimension too small");
    Scratch sc(ctx);
    double *G = nullptr, *lam = nullptr, *vecs = nullptr;
    float* Wsmall = nullptr;
    PB_TRY(sc.alloc(&G, (size_t)c * c));
    PB_TRY(sc.alloc(&lam, (size_t)c));
    PB_TRY(sc.alloc(&vecs, (size_t)c * c));
    PB_TRY(sc.alloc(&Wsmall, (size_t)c * rank));
    PB_TRY(pb_gram(ctx, M, n, c, ldm, G));
    PB_TRY(pb_reduce(ctx, G, (int64_t)c * c, PB200_F64));     // row-sharded M (reduce hook installed): global Gram matrix
    PB_TRY(pb_eig_psd(ctx, G, c, lam, vecs));
    sqrt_leading_kernel<<<(rank + 127) / 128, 128, 0, ctx->stream>>>(lam, rank, sigma_out);
    take_columns_kernel<<<(c * rank + 255) / 256, 256, 0, ctx->stream>>>(vecs, c, rank, lam, 1, Wsmall);
    PB_TRY(pb_right_multiply(ctx, M, n, c, ldm, Wsmall, rank, rank, U_out, ldu));
    if (Vt_out) rows_to_float_kernel<<<(c * rank + 255) / 256, 256, 0, ctx->stream>>>(vecs, c, rank, Vt_out);
    ctx->stats[0] += 3;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

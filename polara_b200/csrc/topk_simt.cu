// Exact fp32 fused scoring kernel (CUDA cores):  scores = E V^T  ->  seen mask -> top-k,
// one block per (64-user tile, item part); score rows live only in registers.
//
// Replaces, fused: the dgemm of SVDModel.slice_recommendations (polara/recommender/
// models.py:857-861), downvote_seen_items (models.py:494-519) and get_topk_elements
// (models.py:522-564).  This is the reference implementation of the device contract; the
// tensor-core kernel (topk_tc.cu) must produce bit-identical lists.  `id_map` (optional) renames the
// rows of V (used when V is a gathered subset): ids in the lists and seen lookups use id_map[row].
#include "topk_common.cuh"

namespace {

constexpr int TU = 64;     // users per block
constexpr int TI = 128;    // items per step
constexpr int KS = 32;     // k slab
constexpr int ES = TU + 4;
constexpr int VS = TI + 4;

struct SimtSmem {
    float es[KS][ES];
    float vs[KS][VS];
    pb200_cand cand[TU][TI];
    int cnt[TU];
    int lcnt[TU];
    float thr[TU];
};

__global__ void __launch_bounds__(256)
score_topk_simt_kernel(const float* __restrict__ E, int64_t lde, const float* __restrict__ V, int64_t ldv,
                       int64_t m, int64_t n, int r, const int64_t* __restrict__ seen_indptr,
                       const int32_t* __restrict__ seen_indices, int64_t seen_offset, int k, int parts,
                       pb200_cand* __restrict__ lists, const int32_t* __restrict__ id_map) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SimtSmem& sm = *reinterpret_cast<SimtSmem*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tx = tid & 15, ty = tid >> 4;
    const int64_t u0 = (int64_t)blockIdx.x * TU;
    const int part = blockIdx.y;
    const int64_t tiles_total = (n + TI - 1) / TI;
    const int64_t tiles_per_part = (tiles_total + parts - 1) / parts;
    const int64_t item_lo = min(n, (int64_t)part * tiles_per_part * TI);
    const int64_t item_hi = min(n, (int64_t)(part + 1) * tiles_per_part * TI);

    for (int u = tid; u < TU; u += 256) { sm.cnt[u] = 0; sm.lcnt[u] = 0; sm.thr[u] = -CUDART_INF_F; }
    // every (part, user) list is fully initialised here
    for (int64_t e = tid; e < (int64_t)TU * k; e += 256) {
        int64_t u = u0 + e / k;
        if (u < m) { pb200_cand c; c.score = -CUDART_INF_F; c.id = -1; lists[((int64_t)part * m + u) * k + e % k] = c; }
    }
    __syncthreads();

    for (int64_t i0 = item_lo; i0 < item_hi; i0 += TI) {
        float acc[4][8];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 8; ++b) acc[a][b] = 0.f;
        for (int k0 = 0; k0 < r; k0 += KS) {
#pragma unroll
            for (int it = 0; it < 8; ++it) {
                int e = tid + it * 256;
                int row = e >> 5, kk = e & 31;
                int64_t u = u0 + row;
                float v = 0.f;
                if (u < m && k0 + kk < r) v = __ldg(E + u * lde + k0 + kk);
                sm.es[kk][row] = v;
            }
#pragma unroll
            for (int it = 0; it < 16; ++it) {
                int e = tid + it * 256;
                int row = e >> 5, kk = e & 31;
                int64_t j = i0 + row;
                float v = 0.f;
                if (j < item_hi && k0 + kk < r) v = __ldg(V + j * ldv + k0 + kk);
                sm.vs[kk][row] = v;
            }
            __syncthreads();
            const int kmax = min(KS, r - k0);
            for (int kk = 0; kk < kmax; ++kk) {
                float4 e4 = *reinterpret_cast<const float4*>(&sm.es[kk][ty * 4]);
                float4 v0 = *reinterpret_cast<const float4*>(&sm.vs[kk][tx * 8]);
                float4 v1 = *reinterpret_cast<const float4*>(&sm.vs[kk][tx * 8 + 4]);
                float a[4] = {e4.x, e4.y, e4.z, e4.w};
                float b[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
            }
            __syncthreads();
        }
        // ---- candidate filter: anything not worse than the current k-th score ----
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int ul = ty * 4 + i;
            if (u0 + ul >= m) continue;
            float th = sm.thr[ul];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                int64_t item = i0 + tx * 8 + j;
                if (item < item_hi && acc[i][j] >= th) {
                    int slot = atomicAdd(&sm.cnt[ul], 1);
                    pb200_cand c; c.score = acc[i][j]; c.id = id_map ? __ldg(id_map + item) : (int)item;
                    sm.cand[ul][slot] = c;
                }
            }
        }
        __syncthreads();
        // ---- merge candidates into the per-user lists (one warp per user) ----
        for (int ul = warp; ul < TU; ul += 8) {
            int nc = sm.cnt[ul];
            if (nc == 0) continue;
            int64_t u = u0 + ul;
            if (seen_indptr) {
                int64_t sb = seen_indptr[u], se = seen_indptr[u + 1];
                for (int c = lane; c < nc; c += 32) {
                    if (seen_lookup(seen_indices, sb, se, (int)(sm.cand[ul][c].id + seen_offset))) sm.cand[ul][c].id = -1;
                }
                __syncwarp();
            }
            pb200_cand* list = lists + ((int64_t)part * m + u) * k;
            int lc = sm.lcnt[ul];
            for (int c = 0; c < nc; ++c) {
                pb200_cand cd = sm.cand[ul][c];
                if (cd.id < 0) continue;
                lc = warp_list_insert(list, k, lc, cd.score, cd.id, lane);
            }
            __syncwarp();
            if (lane == 0) {
                sm.lcnt[ul] = lc;
                sm.cnt[ul] = 0;
                sm.thr[ul] = (lc == k) ? list[k - 1].score : -CUDART_INF_F;
            }
        }
        __syncthreads();
    }
}

}  // namespace

int pb_score_simt(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv, int64_t m,
                  int64_t n, int r, const int64_t* seen_indptr, const int32_t* seen_indices, int64_t seen_offset,
                  int k, int parts, pb200_cand* lists, const int32_t* id_map) {
    if (m == 0) return PB200_OK;
    // the attribute is per device (a process may hold one context per device): set it on every call, it is cheap
    PB_CUDA(ctx, cudaFuncSetAttribute(score_topk_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)sizeof(SimtSmem)));
    dim3 grid((unsigned)ceil_div64(m, TU), (unsigned)parts);
    cudaEventRecord(ctx->ev0, ctx->stream);
    score_topk_simt_kernel<<<grid, 256, sizeof(SimtSmem), ctx->stream>>>(E, lde, V, ldv, m, n, r, seen_indptr,
                                                                         seen_indices, seen_offset, k, parts, lists, id_map);
    cudaEventRecord(ctx->ev1, ctx->stream);
    ctx->stats[0] += 1;
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

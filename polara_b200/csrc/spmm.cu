// CSR SpMM  Y[n_rows x ell] (+)= A * X  (fp32), deterministic (fixed summation order, no float atomics).
//
// Replaces csr_matrix.dot(ndarray) (polara/recommender/models.py:860) and the
// A x / A^T x products inside scipy.sparse.linalg.svds (models.py:844).
//
// Main kernel (spmm_stage_kernel) -- dense rows of X are STAGED IN SHARED MEMORY by bulk async copies:
//   * work split by NNZ, not by rows: block b owns the nnz window [b*CB, (b+1)*CB) of the matrix (or of one column
//     panel of it), so a popular item's 1e6-nnz row in A^T is spread over ~500 blocks instead of one;
//   * warp 0 (producer): lanes read 32 column ids coalesced and each issues ONE cp.async.bulk of the X row segment
//     (128*LPT bytes) into a ring of slots in shared memory; mbarrier complete_tx tracks every group of 32 rows.
//     X gathers carry an L2 evict_last policy, the streamed (col, val) arrays evict_first, so the dense panel stays
//     L2-resident while the matrix streams through;
//   * warps 1..LPT (consumers): warp j owns columns [32j, 32j+32) and walks all nnz of the window in order: 32 staged
//     values -> registers (conflict-free LDS), one FMA per nnz, values broadcast by shuffle; at a row boundary the
//     accumulator goes to Y (one coalesced 128-byte store per warp);
//   * a row that straddles window boundaries: the block where it STARTS writes its piece to Y, every later piece goes
//     to carry[b]; spmm_fixup_kernel adds the carries of a row in block order (fixed order => deterministic).
//   * column panels (pb200_csr_block_columns): when X is larger than L2 (A^T W with 1e6 users: 384 MB) the matrix is
//     stored panel-major (virtual row = panel * n_rows + row) with panels of X rows sized to stay L2-resident; panels
//     are launched one after another and accumulate into Y in panel order.
// Algorithmic bytes: 8*nnz + 8*(rows+1) + 4*ell*(cols + rows); the per-nnz gather of X rows (nnz*ell*4 B) is L2 traffic.
//
// Fallback (spmm_ldg_kernel): register gathers with __ldg for operands that do not meet the 16-byte alignment rules of
// the bulk copies (ldx % 4 != 0, unaligned base); same window/carry scheme is not needed there (row-owned).
#include "common.cuh"

namespace {

// ------------------------------------------------------------------------------------------------------------------
//  fallback: row-owned register-gather kernel (round-1 kernel)
// ------------------------------------------------------------------------------------------------------------------
constexpr int CB = 2048;        // nnz window per block
constexpr int WARPS = 8;
constexpr int LONG_ROW = 4096;  // rows longer than this are processed by the whole block
constexpr int MAX_LONG = CB / LONG_ROW + 2;

__device__ __forceinline__ int64_t lower_bound_i64(const int64_t* a, int64_t n, int64_t key) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (a[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

template <int LPT>
__device__ __forceinline__ void accumulate_range(float (&acc)[LPT], int64_t beg, int64_t end,
                                                 int64_t step_batches, const int32_t* __restrict__ indices,
                                                 const float* __restrict__ values,
                                                 const float* __restrict__ X, int64_t ldx, int lane, int live) {
    // columns >= live are padding: their lanes neither load nor accumulate
    bool on[LPT];
#pragma unroll
    for (int j = 0; j < LPT; ++j) on[j] = lane + 32 * j < live;
    for (int64_t p = beg; p < end; p += 32 * step_batches) {
        int64_t q = p + lane;
        int32_t c = 0;
        float v = 0.f;
        if (q < end) { c = __ldg(indices + q); v = __ldg(values + q); }
        int cnt = (int)min((int64_t)32, end - p);
        for (int t = 0; t < cnt; ++t) {
            int32_t c0 = __shfl_sync(0xffffffffu, c, t);
            float v0 = __shfl_sync(0xffffffffu, v, t);
            const float* x0 = X + (int64_t)c0 * ldx + lane;
#pragma unroll
            for (int j = 0; j < LPT; ++j) acc[j] = fmaf(v0, on[j] ? __ldg(x0 + 32 * j) : 0.f, acc[j]);
        }
    }
}

template <int LPT>
__global__ void __launch_bounds__(WARPS * 32)
spmm_ldg_kernel(int64_t n_rows, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                const float* __restrict__ values, const float* __restrict__ X, int64_t ldx, float* __restrict__ Y,
                int64_t ldy, int64_t nnz_begin, int64_t n_blocks, int live, int accumulate) {
    __shared__ int64_t s_rows[2];
    __shared__ int s_next;
    __shared__ int s_nlong;
    __shared__ int64_t s_long[MAX_LONG];
    __shared__ float s_part[WARPS][32 * LPT];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t b = blockIdx.x;
    if (threadIdx.x == 0) {
        // rows whose FIRST nnz position lies in this block's window (empty rows go with the pointer they sit at)
        s_rows[0] = b == 0 ? 0 : lower_bound_i64(indptr, n_rows, nnz_begin + b * (int64_t)CB);
        s_rows[1] = (b == n_blocks - 1) ? n_rows : lower_bound_i64(indptr, n_rows, nnz_begin + (b + 1) * (int64_t)CB);
        s_next = 0;
        s_nlong = 0;
    }
    __syncthreads();
    const int64_t row_lo = s_rows[0], row_hi = s_rows[1];
    for (;;) {
        int idx = 0;
        if (lane == 0) idx = atomicAdd(&s_next, 1);
        idx = __shfl_sync(0xffffffffu, idx, 0);
        int64_t row = row_lo + idx;
        if (row >= row_hi) break;
        int64_t beg = indptr[row], end = indptr[row + 1];
        if (end - beg > LONG_ROW) {
            if (lane == 0) { int s = atomicAdd(&s_nlong, 1); if (s < MAX_LONG) s_long[s] = row; }
            continue;
        }
        float acc[LPT];
#pragma unroll
        for (int j = 0; j < LPT; ++j) acc[j] = 0.f;
        accumulate_range<LPT>(acc, beg, end, 1, indices, values, X, ldx, lane, live);
        float* y = Y + row * ldy + lane;
#pragma unroll
        for (int j = 0; j < LPT; ++j) y[32 * j] = accumulate ? y[32 * j] + acc[j] : acc[j];
    }
    __syncthreads();
    const int nlong = min(s_nlong, MAX_LONG);
    for (int li = 0; li < nlong; ++li) {
        int64_t row = s_long[li];
        int64_t beg = indptr[row], end = indptr[row + 1];
        float acc[LPT];
#pragma unroll
        for (int j = 0; j < LPT; ++j) acc[j] = 0.f;
        accumulate_range<LPT>(acc, beg + 32 * (int64_t)warp, end, WARPS, indices, values, X, ldx, lane, live);
#pragma unroll
        for (int j = 0; j < LPT; ++j) s_part[warp][lane + 32 * j] = acc[j];
        __syncthreads();
        if (warp == 0) {
#pragma unroll
            for (int j = 0; j < LPT; ++j) {
                float s = 0.f;
                for (int w = 0; w < WARPS; ++w) s += s_part[w][lane + 32 * j];
                float* y = Y + row * ldy + lane + 32 * j;
                *y = accumulate ? *y + s : s;
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------------------------
//  main: shared-memory staged kernel
// ------------------------------------------------------------------------------------------------------------------
constexpr int SB = 2048;                      // nnz per block window (multiple of 32)
constexpr int GROUP = 32;                     // nnz per ring group = one mbarrier phase
constexpr long long SPIN_LIMIT = 4000000000ll;   // ~2 s: never hang the GPU, trap instead

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%1], %0;" ::"r"(count), "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%1], %0;" ::"r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred P1;\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\tselp.b32 %0, 1, 0, P1;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __noinline__ void mbar_wait_slow(uint32_t bar, uint32_t parity, unsigned long long* stats) {
    uint32_t spins = 0;
    long long t_start = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0xFFFu) == 0) {
            long long now = clock64();
            if (t_start == 0) t_start = now;
            else if (now - t_start > SPIN_LIMIT) {
                if (stats) atomicExch(stats + 7, 0x5B3D0000ull | (bar & 0xFFFFu));
                asm volatile("trap;");
            }
        }
    }
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, unsigned long long* stats) {
    if (mbar_try_wait(bar, parity)) return;
    mbar_wait_slow(bar, parity, stats);
}
__device__ __forceinline__ uint64_t policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
// warp-uniform form: every lane passes the SAME operands, one elected lane issues (no per-lane waterfall loop around
// UBLKCP, whose operands live in uniform registers)
__device__ __forceinline__ void bulk_g2s_hint_elect(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t pol) {
    asm volatile("{\n\t.reg .pred q;\n\telect.sync _|q, 0xffffffff;\n\t"
                 "@q cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;\n\t}"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async16_hint(uint32_t dst, const void* src, uint64_t pol) {
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint32_t bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ int32_t ld_stream_i32(const int32_t* p, uint64_t pol) {
    int32_t v;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ float ld_stream_f32(const float* p, uint64_t pol) {
    float v;
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol));
    return v;
}

// first r in [0, n] with a[r] >= key  (a has n+1 entries, non-decreasing)
__device__ __forceinline__ int64_t lower_bound_ptr(const int64_t* __restrict__ a, int64_t n, int64_t key) {
    int64_t lo = 0, hi = n + 1;
    while (lo < hi) {
        int64_t mid = (lo + hi) >> 1;
        if (__ldg(a + mid) < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// the same result from a whole warp: each step 32 lanes probe 32 evenly spaced pointers, so 1M rows take 4 dependent
// loads instead of 20
__device__ __forceinline__ int64_t lower_bound_ptr_warp(const int64_t* __restrict__ a, int64_t n, int64_t key, int lane) {
    int64_t lo = 0, hi = n + 1;                          // answer in [lo, hi]; a[hi] >= key or hi == n + 1
    while (hi - lo > 32) {
        const int64_t s = (hi - lo + 31) >> 5;
        const int64_t q = min(lo + (lane + 1) * s, hi) - 1;
        const uint32_t ge = __ballot_sync(0xffffffffu, __ldg(a + q) >= key);
        if (ge == 0) return hi;
        const int f = __ffs(ge) - 1;
        hi = min(lo + (f + 1) * s, hi) - 1;
        lo = lo + f * s;
    }
    const uint32_t ge = __ballot_sync(0xffffffffu, lo + lane < hi && __ldg(a + lo + lane) >= key);
    return ge ? lo + __ffs(ge) - 1 : hi;
}

// LPT  = 32-column groups per row segment (1..4); warp j of the consumers owns columns [32j, 32j+32).
// NG   = ring depth in groups of 32 staged rows (staged variants).
// PROD = 0: X rows staged in shared memory by cp.async.bulk (UBLKCP), one bulk copy per row, complete_tx on an mbarrier;
//        1: staged by 16-byte cp.async (LDGSTS) chunks, the producer lanes arrive on the mbarrier when their copies landed.
// (Gathering straight into registers lives in spmm_window*_kernel below.)
// In every variant the window's (column id, value) pairs are first copied to shared memory by the whole block, so the
// DRAM latency of the streamed arrays is paid once per window instead of once per group of 32 nnz.
template <int LPT, int NG, int PROD>
__global__ void __launch_bounds__(32 * (LPT + 1))
spmm_stage_kernel(int64_t n_rows, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                  const float* __restrict__ values, const float* __restrict__ X, int64_t ldx,
                  float* __restrict__ Y, int64_t ldy, int64_t nnz_begin, int64_t nnz_end, int64_t n_blocks,
                  int live /* columns of this launch that exist, 1..32*LPT */, uint32_t copy_bytes, int accumulate,
                  float* __restrict__ carry /*[n_blocks][32*LPT]*/, int64_t* __restrict__ carry_row /*[n_blocks]*/,
                  unsigned long long* stats) {
    constexpr int SLOT = 128 * LPT;                      // bytes
    constexpr int NPROD = 1;                             // producer warps
    extern __shared__ __align__(128) unsigned char ring[];   // [NG][GROUP][SLOT]   (staged variants)
    __shared__ int32_t s_idx[SB];
    __shared__ float s_val[SB];
    __shared__ __align__(8) uint64_t bars[2 * NG];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + NG);
    const int64_t b = blockIdx.x;
    const int64_t w0 = nnz_begin + b * (int64_t)SB;
    const int64_t w1 = min(nnz_end, w0 + SB);
    const int rel_w1 = (int)max(w1 - w0, (int64_t)0);
    const int n_groups = (rel_w1 + GROUP - 1) / GROUP;
    if (PROD != 2 && threadIdx.x == 0) {
        for (int g = 0; g < NG; ++g) { mbar_init(bar_full + 8 * g, PROD == 0 ? 1 : 32); mbar_init(bar_empty + 8 * g, LPT); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    {
        // the window's streamed arrays -> shared memory (coalesced, evict-first: they are read exactly once)
        const uint64_t pol_stream = policy_evict_first();
        for (int e = threadIdx.x; e < rel_w1; e += blockDim.x) {
            s_idx[e] = ld_stream_i32(indices + w0 + e, pol_stream);
            s_val[e] = ld_stream_f32(values + w0 + e, pol_stream);
        }
    }
    __syncthreads();

    if (PROD != 2 && warp == 0) {
        // ================================ producer =================================================================
        const uint64_t pol_keep = policy_evict_last();
        const uint32_t ring0 = smem_u32(ring);
        for (int i = 0; i < n_groups; ++i) {
            const int g = i % NG;
            const uint32_t ph = (uint32_t)(i / NG) & 1u;
            const int rel0 = i * GROUP;
            const int cnt = min(GROUP, rel_w1 - rel0);
            const int32_t c = lane < cnt ? s_idx[rel0 + lane] : 0;
            mbar_wait(bar_empty + 8 * g, ph ^ 1u, stats);            // consumers are done with the previous tenant
            if constexpr (PROD == 0) {
                if (lane == 0) mbar_arrive_expect_tx(bar_full + 8 * g, (uint32_t)cnt * copy_bytes);
                __syncwarp();
#pragma unroll
                for (int t = 0; t < GROUP; ++t) {
                    const int32_t ct = __shfl_sync(0xffffffffu, c, t);
                    if (t < cnt)
                        bulk_g2s_hint_elect(ring0 + (uint32_t)((g * GROUP + t) * SLOT), X + (int64_t)ct * ldx, copy_bytes,
                                            bar_full + 8 * g, pol_keep);
                }
            } else {
                const int cpc = (int)(copy_bytes >> 4);                 // 16-byte chunks per staged row
                const int total = cnt * cpc;
                for (int e = lane; e < ((total + 31) & ~31); e += 32) {
                    const int slot_i = e / cpc, ch = e - slot_i * cpc;
                    const int32_t ct = __shfl_sync(0xffffffffu, c, slot_i & 31);
                    if (e < total)
                        cp_async16_hint(ring0 + (uint32_t)((g * GROUP + slot_i) * SLOT + ch * 16),
                                        reinterpret_cast<const unsigned char*>(X + (int64_t)ct * ldx) + ch * 16, pol_keep);
                }
                cp_async_mbar_arrive_noinc(bar_full + 8 * g);            // fires when this lane's copies have landed
            }
        }
    } else {
        // ================================ consumers ================================================================
        const int j = warp - NPROD;                      // column group of this warp
        const int col = 32 * j + lane;
        const bool col_live = col < live;
        // ---- which rows does the window touch?  (runs while the first copies are in flight) -----------------------
        // rows are OWNED by the block whose window holds their first nnz position (empty rows: the pointer they sit at;
        // the last block also owns pointer == nnz_end)
        const int64_t own_end = (b == n_blocks - 1) ? nnz_end + 1 : w1;
        int64_t cur;
        bool piece_is_carry;
        {
            const int64_t lb = b == 0 ? 0 : lower_bound_ptr(indptr, n_rows, w0);     // first row with indptr >= w0
            if (lb <= n_rows && (b == 0 || __ldg(indptr + lb) == w0)) { cur = lb; piece_is_carry = false; }
            else { cur = lb - 1; piece_is_carry = true; }                             // a row that began before w0
        }
        if (lane == 0 && j == 0) carry_row[b] = piece_is_carry ? cur : -1;
        // lane t holds (indptr[pbase + t] - w0), clamped to the int32 range of the window
        int64_t pbase = cur;
        auto load_ptrs = [&](int64_t base) -> int {
            const int64_t r = min(base + lane, n_rows);
            const int64_t v = __ldg(indptr + r) - w0;
            return (int)max((int64_t)-1, min(v, (int64_t)SB + 2));
        };
        int ptrs = load_ptrs(pbase);
        auto row_end_rel = [&]() -> int {                // end of row `cur` relative to w0 (clamped)
            if (cur + 1 - pbase >= 32) { pbase = cur; ptrs = load_ptrs(pbase); }
            return __shfl_sync(0xffffffffu, ptrs, (int)(cur + 1 - pbase));
        };
        auto emit = [&](float acc, bool empty_row) {
            if (piece_is_carry) carry[b * (int64_t)(32 * LPT) + col] = acc;
            else if (!accumulate) Y[cur * ldy + col] = acc;
            else if (!empty_row) { float* y = Y + cur * ldy + col; *y = *y + acc; }
            piece_is_carry = false;
        };
        float acc = 0.f;
        int rel_end = row_end_rel();
        bool touched = false;                            // has the current row received an nnz in this window?
        const int rel_own = (int)(own_end - w0);
        // one group of 32 nnz: x[t] = X[col of nnz t][this lane's column]; v = this lane's nnz value
        auto sweep = [&](const float (&x)[GROUP], float v, int rel0, int cnt) {
#pragma unroll
            for (int t = 0; t < GROUP; ++t) {
                if (t < cnt) {
                    while (rel0 + t == rel_end) {                    // row `cur` ends before this nnz (empty rows loop)
                        emit(acc, !touched);
                        acc = 0.f;
                        touched = false;
                        ++cur;
                        rel_end = row_end_rel();
                    }
                    acc = fmaf(__shfl_sync(0xffffffffu, v, t), x[t], acc);
                    touched = true;
                }
            }
        };
        {
            for (int i = 0; i < n_groups; ++i) {
                const int g = i % NG;
                const uint32_t ph = (uint32_t)(i / NG) & 1u;
                const int rel0 = i * GROUP;
                const int cnt = min(GROUP, rel_w1 - rel0);
                const float v = lane < cnt ? s_val[rel0 + lane] : 0.f;
                mbar_wait(bar_full + 8 * g, ph, stats);
                float x[GROUP];
                const float* slot = reinterpret_cast<const float*>(ring + (size_t)g * GROUP * SLOT) + col;
#pragma unroll
                for (int t = 0; t < GROUP; ++t) x[t] = (t < cnt && col_live) ? slot[t * (SLOT / 4)] : 0.f;
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_empty + 8 * g);       // values are in registers: the slots may be refilled
                sweep(x, v, rel0, cnt);
            }
        }
        // ---- window exhausted.  Row `cur` holds the last nnz of the window (or, in an empty window, sits at the
        // window's pointer): its piece is complete or continues in the next block -- either way it is written now.
        // After it, rows that BEGIN before own_end are empty rows at the end pointer (last block / empty matrix).
        emit(acc, !touched);
        while (rel_end < rel_own) {
            ++cur;
            if (cur >= n_rows) break;
            rel_end = row_end_rel();
            emit(0.f, true);
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
//  nnz windows per WARP + register gathers: the default.  Every warp owns a window of SW consecutive nnz (of the matrix
//  or of one column panel) and ALL 32*LPT columns of the launch: per nnz 2 shuffles + LPT coalesced 128-byte gathers +
//  LPT FMAs, four nnz in flight, no row-boundary test inside a row segment.  Same ownership / carry rules as above.
// ------------------------------------------------------------------------------------------------------------------
constexpr int SW = 1024;                      // nnz per warp window (multiple of 32)
constexpr int WWARPS = 8;                     // warps per block

template <int LPT>
__global__ void __launch_bounds__(WWARPS * 32)
spmm_window_kernel(int64_t n_rows, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                   const float* __restrict__ values, const float* __restrict__ X, int64_t ldx,
                   float* __restrict__ Y, int64_t ldy, int64_t nnz_begin, int64_t nnz_end, int64_t n_windows,
                   int live, int accumulate, float* __restrict__ carry /*[n_windows][32*LPT]*/,
                   int64_t* __restrict__ carry_row /*[n_windows]*/) {
    const int lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * WWARPS + (threadIdx.x >> 5);      // window index
    if (b >= n_windows) return;
    const int64_t w0 = nnz_begin + b * (int64_t)SW;
    const int64_t w1 = min(nnz_end, w0 + SW);
    const int rel_w1 = (int)max(w1 - w0, (int64_t)0);
    const int n_groups = (rel_w1 + 31) / 32;
    const uint64_t pol_stream = policy_evict_first();
    bool on[LPT];
#pragma unroll
    for (int j = 0; j < LPT; ++j) on[j] = lane + 32 * j < live;
    // first group of (col, val) is requested before the row search so that both latencies overlap
    int32_t c_next = 0;
    float v_next = 0.f;
    if (lane < rel_w1) { c_next = ld_stream_i32(indices + w0 + lane, pol_stream); v_next = ld_stream_f32(values + w0 + lane, pol_stream); }
    const int64_t own_end = (b == n_windows - 1) ? nnz_end + 1 : w1;
    int64_t cur;
    bool piece_is_carry;
    {
        const int64_t lb = b == 0 ? 0 : lower_bound_ptr(indptr, n_rows, w0);
        if (lb <= n_rows && (b == 0 || __ldg(indptr + lb) == w0)) { cur = lb; piece_is_carry = false; }
        else { cur = lb - 1; piece_is_carry = true; }
    }
    if (lane == 0) carry_row[b] = piece_is_carry ? cur : -1;
    int64_t pbase = cur;
    auto load_ptrs = [&](int64_t base) -> int {
        const int64_t r = min(base + lane, n_rows);
        const int64_t v = __ldg(indptr + r) - w0;
        return (int)max((int64_t)-1, min(v, (int64_t)SW + 2));
    };
    int ptrs = load_ptrs(pbase);
    auto row_end_rel = [&]() -> int {
        if (cur + 1 - pbase >= 32) { pbase = cur; ptrs = load_ptrs(pbase); }
        return __shfl_sync(0xffffffffu, ptrs, (int)(cur + 1 - pbase));
    };
    float acc[LPT];
#pragma unroll
    for (int j = 0; j < LPT; ++j) acc[j] = 0.f;
    auto emit = [&](bool empty_row) {
        if (piece_is_carry) {
#pragma unroll
            for (int j = 0; j < LPT; ++j) carry[b * (int64_t)(32 * LPT) + lane + 32 * j] = acc[j];
        } else if (!accumulate) {
#pragma unroll
            for (int j = 0; j < LPT; ++j) Y[cur * ldy + lane + 32 * j] = acc[j];
        } else if (!empty_row) {
#pragma unroll
            for (int j = 0; j < LPT; ++j) { float* y = Y + cur * ldy + lane + 32 * j; *y = *y + acc[j]; }
        }
        piece_is_carry = false;
#pragma unroll
        for (int j = 0; j < LPT; ++j) acc[j] = 0.f;
    };
    int rel_end = row_end_rel();
    bool touched = false;
    const int rel_own = (int)(own_end - w0);
    const float* xl = X + lane;
    for (int i = 0; i < n_groups; ++i) {
        const int rel0 = i * 32;
        const int cnt = min(32, rel_w1 - rel0);
        const int32_t c = c_next;
        const float v = v_next;
        if (rel0 + 32 + lane < rel_w1) {
            c_next = ld_stream_i32(indices + w0 + rel0 + 32 + lane, pol_stream);
            v_next = ld_stream_f32(values + w0 + rel0 + 32 + lane, pol_stream);
        }
        int t = 0;
        while (t < cnt) {
            while (rel0 + t == rel_end) {                        // rows that end here (empty rows loop)
                emit(!touched);
                touched = false;
                ++cur;
                rel_end = row_end_rel();
            }
            const int seg_end = min(cnt, rel_end - rel0);        // the current row owns nnz [t, seg_end) of this group
            for (; t + 4 <= seg_end; t += 4) {
                const int32_t c0 = __shfl_sync(0xffffffffu, c, t), c1 = __shfl_sync(0xffffffffu, c, t + 1);
                const int32_t c2 = __shfl_sync(0xffffffffu, c, t + 2), c3 = __shfl_sync(0xffffffffu, c, t + 3);
                const float v0 = __shfl_sync(0xffffffffu, v, t), v1 = __shfl_sync(0xffffffffu, v, t + 1);
                const float v2 = __shfl_sync(0xffffffffu, v, t + 2), v3 = __shfl_sync(0xffffffffu, v, t + 3);
                const float* x0 = xl + (int64_t)c0 * ldx;
                const float* x1 = xl + (int64_t)c1 * ldx;
                const float* x2 = xl + (int64_t)c2 * ldx;
                const float* x3 = xl + (int64_t)c3 * ldx;
                float a0[LPT], a1[LPT], a2[LPT], a3[LPT];
#pragma unroll
                for (int j = 0; j < LPT; ++j) {
                    a0[j] = on[j] ? __ldg(x0 + 32 * j) : 0.f; a1[j] = on[j] ? __ldg(x1 + 32 * j) : 0.f;
                    a2[j] = on[j] ? __ldg(x2 + 32 * j) : 0.f; a3[j] = on[j] ? __ldg(x3 + 32 * j) : 0.f;
                }
#pragma unroll
                for (int j = 0; j < LPT; ++j) {
                    acc[j] = fmaf(v0, a0[j], acc[j]); acc[j] = fmaf(v1, a1[j], acc[j]);
                    acc[j] = fmaf(v2, a2[j], acc[j]); acc[j] = fmaf(v3, a3[j], acc[j]);
                }
            }
            for (; t < seg_end; ++t) {
                const int32_t c0 = __shfl_sync(0xffffffffu, c, t);
                const float v0 = __shfl_sync(0xffffffffu, v, t);
                const float* x0 = xl + (int64_t)c0 * ldx;
#pragma unroll
                for (int j = 0; j < LPT; ++j) acc[j] = fmaf(v0, on[j] ? __ldg(x0 + 32 * j) : 0.f, acc[j]);
            }
            touched = true;
        }
    }
    emit(!touched);
    while (rel_end < rel_own) {
        ++cur;
        if (cur >= n_rows) break;
        rel_end = row_end_rel();
        emit(true);
    }
}

// Same scheme with 128-bit gathers: a lane owns FOUR consecutive columns, so one LDG.128 per lane covers a whole row segment
// of 64 columns with half a warp (two nnz per instruction; the halves are added when the row is written) or of 128 columns
// with a full warp.  The scalar kernel above spends 78 % of its issue slots; per nnz this one issues about half as many
// instructions.  Needs 16-byte aligned rows (ldx % 4 == 0, aligned base, ldx >= ell rounded up to 4).
template <bool WIDE>
__global__ void __launch_bounds__(WWARPS * 32)
spmm_window4_kernel(int64_t n_rows, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                    const float* __restrict__ values, const float* __restrict__ X, int64_t ldx,
                    float* __restrict__ Y, int64_t ldy, int64_t nnz_begin, int64_t nnz_end, int64_t n_windows,
                    int live, int accumulate, float* __restrict__ carry /*[n_windows][WIDTH]*/,
                    int64_t* __restrict__ carry_row /*[n_windows]*/) {
    constexpr int WIDTH = WIDE ? 128 : 64;
    const int lane = threadIdx.x & 31;
    const int hw = WIDE ? 0 : (lane >> 4);               // which nnz of a pair this half-warp takes
    const int col = WIDE ? 4 * lane : 4 * (lane & 15);   // first of this lane's four columns
    const int64_t b = (int64_t)blockIdx.x * WWARPS + (threadIdx.x >> 5);
    if (b >= n_windows) return;
    const int64_t w0 = nnz_begin + b * (int64_t)SW;
    const int64_t w1 = min(nnz_end, w0 + SW);
    const int rel_w1 = (int)max(w1 - w0, (int64_t)0);
    const int n_groups = (rel_w1 + 31) / 32;
    const uint64_t pol_stream = policy_evict_first();
    const bool st_on = col < ((live + 31) & ~31) && hw == 0;   // Y is written in whole groups of 32 columns
    // columns at or beyond `live` are masked when a row is WRITTEN, not per gather: a lane without live columns repeats
    // the address of the last live lane (same sector, no extra traffic), a partly live lane reads the padding that
    // ldx >= live rounded up to 4 guarantees -- both accumulate values nobody stores
    const bool m0 = col < live, m1 = col + 1 < live, m2 = col + 2 < live, m3 = col + 3 < live;
    int32_t c_next = 0;
    float v_next = 0.f;
    if (lane < rel_w1) { c_next = ld_stream_i32(indices + w0 + lane, pol_stream); v_next = ld_stream_f32(values + w0 + lane, pol_stream); }
    const int64_t own_end = (b == n_windows - 1) ? nnz_end + 1 : w1;
    int64_t cur;
    bool piece_is_carry;
    {
        const int64_t lb = b == 0 ? 0 : lower_bound_ptr_warp(indptr, n_rows, w0, lane);
        if (lb <= n_rows && (b == 0 || __ldg(indptr + lb) == w0)) { cur = lb; piece_is_carry = false; }
        else { cur = lb - 1; piece_is_carry = true; }
    }
    if (lane == 0) carry_row[b] = piece_is_carry ? cur : -1;
    int64_t pbase = cur;
    auto load_ptrs = [&](int64_t base) -> int {
        const int64_t r = min(base + lane, n_rows);
        const int64_t v = __ldg(indptr + r) - w0;
        return (int)max((int64_t)-1, min(v, (int64_t)SW + 2));
    };
    int ptrs = load_ptrs(pbase);
    auto row_end_rel = [&]() -> int {
        if (cur + 1 - pbase >= 32) { pbase = cur; ptrs = load_ptrs(pbase); }
        return __shfl_sync(0xffffffffu, ptrs, (int)(cur + 1 - pbase));
    };
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    auto emit = [&](bool empty_row) {
        float4 tot = acc;
        if (!WIDE) {                                      // even-nnz half + odd-nnz half (a + b == b + a bitwise)
            tot.x += __shfl_xor_sync(0xffffffffu, acc.x, 16); tot.y += __shfl_xor_sync(0xffffffffu, acc.y, 16);
            tot.z += __shfl_xor_sync(0xffffffffu, acc.z, 16); tot.w += __shfl_xor_sync(0xffffffffu, acc.w, 16);
        }
        if (!m0) tot.x = 0.f;
        if (!m1) tot.y = 0.f;
        if (!m2) tot.z = 0.f;
        if (!m3) tot.w = 0.f;
        if (st_on) {
            if (piece_is_carry) *reinterpret_cast<float4*>(carry + b * (int64_t)WIDTH + col) = tot;
            else {
                float4* y = reinterpret_cast<float4*>(Y + cur * ldy + col);
                if (!accumulate) *y = tot;
                else if (!empty_row) { float4 o = *y; o.x += tot.x; o.y += tot.y; o.z += tot.z; o.w += tot.w; *y = o; }
            }
        }
        piece_is_carry = false;
        acc = make_float4(0.f, 0.f, 0.f, 0.f);
    };
    int rel_end = row_end_rel();
    bool touched = false;
    const int rel_own = (int)(own_end - w0);
    // one 32 x 32 -> 64 bit multiply-add per address: column ids are non-negative and a row of X is shorter than 4 GB
    // (the launcher checks ldx < 2^30)
    const char* xl = reinterpret_cast<const char*>(X + min(col, ((live - 1) >> 2) << 2));
    const uint32_t ldb = (uint32_t)ldx * 4u;
    constexpr int STEP = WIDE ? 1 : 2;                    // nnz per gather instruction
    auto gather = [&](int32_t cc) -> float4 {
        uint64_t off;
        asm("mul.wide.u32 %0, %1, %2;" : "=l"(off) : "r"((uint32_t)cc), "r"(ldb));
        return __ldg(reinterpret_cast<const float4*>(xl + off));
    };
    for (int i = 0; i < n_groups; ++i) {
        const int rel0 = i * 32;
        const int cnt = min(32, rel_w1 - rel0);
        const int32_t c = c_next;
        const float v = v_next;
        if (rel0 + 32 + lane < rel_w1) {
            c_next = ld_stream_i32(indices + w0 + rel0 + 32 + lane, pol_stream);
            v_next = ld_stream_f32(values + w0 + rel0 + 32 + lane, pol_stream);
        }
        int t = 0;
        while (t < cnt) {
            while (rel0 + t == rel_end) {
                emit(!touched);
                touched = false;
                ++cur;
                rel_end = row_end_rel();
            }
            const int seg_end = min(cnt, rel_end - rel0);
            for (; t + 4 * STEP <= seg_end; t += 4 * STEP) {
                const int i0 = t + hw, i1 = t + STEP + hw, i2 = t + 2 * STEP + hw, i3 = t + 3 * STEP + hw;
                const int32_t c0 = __shfl_sync(0xffffffffu, c, i0), c1 = __shfl_sync(0xffffffffu, c, i1);
                const int32_t c2 = __shfl_sync(0xffffffffu, c, i2), c3 = __shfl_sync(0xffffffffu, c, i3);
                const float v0 = __shfl_sync(0xffffffffu, v, i0), v1 = __shfl_sync(0xffffffffu, v, i1);
                const float v2 = __shfl_sync(0xffffffffu, v, i2), v3 = __shfl_sync(0xffffffffu, v, i3);
                const float4 x0 = gather(c0), x1 = gather(c1), x2 = gather(c2), x3 = gather(c3);
                acc.x = fmaf(v0, x0.x, acc.x); acc.y = fmaf(v0, x0.y, acc.y); acc.z = fmaf(v0, x0.z, acc.z); acc.w = fmaf(v0, x0.w, acc.w);
                acc.x = fmaf(v1, x1.x, acc.x); acc.y = fmaf(v1, x1.y, acc.y); acc.z = fmaf(v1, x1.z, acc.z); acc.w = fmaf(v1, x1.w, acc.w);
                acc.x = fmaf(v2, x2.x, acc.x); acc.y = fmaf(v2, x2.y, acc.y); acc.z = fmaf(v2, x2.z, acc.z); acc.w = fmaf(v2, x2.w, acc.w);
                acc.x = fmaf(v3, x3.x, acc.x); acc.y = fmaf(v3, x3.y, acc.y); acc.z = fmaf(v3, x3.z, acc.z); acc.w = fmaf(v3, x3.w, acc.w);
            }
            if (t < seg_end) {
                // the segment's tail, at most NT gathers per lane: all are issued before the first is consumed, so a
                // tail costs one round trip instead of one per gather.  The gathers are unconditional (a predicated
                // vector load is completed by predicated moves that wait for it): a lane without an nnz of its own
                // repeats the row of the tail's first nnz, which this instruction reads anyway.
                constexpr int NT = 4 - STEP % 2;                      // most gathers of a tail: 3 nnz or 4 pairs
                const int n_tail = (seg_end - t + STEP - 1) / STEP;
                float4 xt[NT];
                float vt[NT];
                bool okt[NT];
#pragma unroll
                for (int j = 0; j < NT; ++j) {
                    const int i0 = t + j * STEP + hw;
                    okt[j] = i0 < seg_end;                             // an odd tail: the second half-warp sits this one out
                    const int src = okt[j] ? i0 : t;
                    vt[j] = __shfl_sync(0xffffffffu, v, src);
                    xt[j] = gather(__shfl_sync(0xffffffffu, c, src));
                }
#pragma unroll
                for (int j = 0; j < NT; ++j) {
                    if (j < n_tail) {
                        const float v0 = okt[j] ? vt[j] : 0.f;
                        const float4 x0 = okt[j] ? xt[j] : make_float4(0.f, 0.f, 0.f, 0.f);
                        acc.x = fmaf(v0, x0.x, acc.x); acc.y = fmaf(v0, x0.y, acc.y); acc.z = fmaf(v0, x0.z, acc.z); acc.w = fmaf(v0, x0.w, acc.w);
                    }
                }
            }
            t = seg_end;
            touched = true;
        }
    }
    emit(!touched);
    while (rel_end < rel_own) {
        ++cur;
        if (cur >= n_rows) break;
        rel_end = row_end_rel();
        emit(true);
    }
}

// adds the carried pieces of every straddling row in block order
__global__ void spmm_fixup_kernel(const float* __restrict__ carry, const int64_t* __restrict__ carry_row, int64_t n_blocks,
                                  float* __restrict__ Y, int64_t ldy, int width, int stride) {
    const int64_t b = blockIdx.x;
    const int64_t r = carry_row[b];
    if (r < 0) return;
    if (b > 0 && carry_row[b - 1] == r) return;          // not the first carried piece of this row
    for (int c = threadIdx.x; c < width; c += blockDim.x) {
        float y = Y[r * ldy + c];
        for (int64_t bb = b; bb < n_blocks && carry_row[bb] == r; ++bb) y += carry[bb * stride + c];
        Y[r * ldy + c] = y;
    }
}

template <int LPT>
constexpr int ring_groups() { return LPT == 1 ? 8 : LPT == 2 ? 6 : LPT == 3 ? 4 : 3; }

template <int LPT>
int launch_stage(pb200_ctx* ctx, int64_t n_rows, const int64_t* indptr, const int32_t* indices, const float* values,
                 const float* X, int64_t ldx, float* Y, int64_t ldy, int64_t nnz_begin, int64_t nnz_end, int live,
                 int accumulate, Scratch& sc) {
    constexpr int NG = ring_groups<LPT>();
    const int prod = ctx->spmm_kernel - 1;              // 0 bulk-staged, 1 cp.async-staged, 2 direct register gathers
    const int64_t n_blocks = std::max<int64_t>(1, ceil_div64(nnz_end - nnz_begin, SB));
    PB_REQUIRE(ctx, n_blocks < (int64_t)2147483647, "spmm: nnz too large for one launch");
    float* carry = nullptr;
    int64_t* carry_row = nullptr;
    PB_TRY(sc.alloc(&carry, (size_t)n_blocks * 32 * LPT));
    PB_TRY(sc.alloc(&carry_row, (size_t)n_blocks));
    const size_t smem = (size_t)NG * GROUP * 128 * LPT;
    const uint32_t copy_bytes = (uint32_t)((live * 4 + 15) / 16 * 16);
#define PB_STAGE_LAUNCH(P, THREADS, SMEM)                                                                                  \
    do {                                                                                                                   \
        PB_CUDA(ctx, cudaFuncSetAttribute(spmm_stage_kernel<LPT, NG, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(SMEM))); \
        spmm_stage_kernel<LPT, NG, P><<<(unsigned)n_blocks, THREADS, SMEM, ctx->stream>>>(                                 \
            n_rows, indptr, indices, values, X, ldx, Y, ldy, nnz_begin, nnz_end, n_blocks, live, copy_bytes, accumulate,   \
            carry, carry_row, reinterpret_cast<unsigned long long*>(ctx->d_stats));                                        \
    } while (0)
    if (prod == 0) PB_STAGE_LAUNCH(0, 32 * (LPT + 1), smem);
    else PB_STAGE_LAUNCH(1, 32 * (LPT + 1), smem);
#undef PB_STAGE_LAUNCH
    spmm_fixup_kernel<<<(unsigned)n_blocks, 32 * LPT, 0, ctx->stream>>>(carry, carry_row, n_blocks, Y, ldy, 32 * LPT, 32 * LPT);
    ctx->stats[0] += 2;
    return PB200_OK;
}

template <int LPT>
int launch_window(pb200_ctx* ctx, int64_t n_rows, const int64_t* indptr, const int32_t* indices, const float* values,
                  const float* X, int64_t ldx, float* Y, int64_t ldy, int64_t nnz_begin, int64_t nnz_end, int live,
                  int accumulate, Scratch& sc) {
    const int64_t n_windows = std::max<int64_t>(1, ceil_div64(nnz_end - nnz_begin, SW));
    const int64_t n_blocks = ceil_div64(n_windows, WWARPS);
    PB_REQUIRE(ctx, n_blocks < (int64_t)2147483647, "spmm: nnz too large for one launch");
    float* carry = nullptr;
    int64_t* carry_row = nullptr;
    PB_TRY(sc.alloc(&carry, (size_t)n_windows * 32 * LPT));
    PB_TRY(sc.alloc(&carry_row, (size_t)n_windows));
    spmm_window_kernel<LPT><<<(unsigned)n_blocks, WWARPS * 32, 0, ctx->stream>>>(n_rows, indptr, indices, values, X, ldx, Y, ldy,
                                                                               nnz_begin, nnz_end, n_windows, live, accumulate,
                                                                               carry, carry_row);
    spmm_fixup_kernel<<<(unsigned)n_windows, 32 * LPT, 0, ctx->stream>>>(carry, carry_row, n_windows, Y, ldy, 32 * LPT, 32 * LPT);
    ctx->stats[0] += 2;
    return PB200_OK;
}

template <bool WIDE>
int launch_window4(pb200_ctx* ctx, int64_t n_rows, const int64_t* indptr, const int32_t* indices, const float* values,
                   const float* X, int64_t ldx, float* Y, int64_t ldy, int64_t nnz_begin, int64_t nnz_end, int live,
                   int accumulate, Scratch& sc) {
    constexpr int WIDTH = WIDE ? 128 : 64;
    const int64_t n_windows = std::max<int64_t>(1, ceil_div64(nnz_end - nnz_begin, SW));
    const int64_t n_blocks = ceil_div64(n_windows, WWARPS);
    PB_REQUIRE(ctx, n_blocks < (int64_t)2147483647, "spmm: nnz too large for one launch");
    float* carry = nullptr;
    int64_t* carry_row = nullptr;
    PB_TRY(sc.alloc(&carry, (size_t)n_windows * WIDTH));
    PB_TRY(sc.alloc(&carry_row, (size_t)n_windows));
    spmm_window4_kernel<WIDE><<<(unsigned)n_blocks, WWARPS * 32, 0, ctx->stream>>>(n_rows, indptr, indices, values, X, ldx, Y, ldy,
                                                                                  nnz_begin, nnz_end, n_windows, live, accumulate,
                                                                                  carry, carry_row);
    const int wlive = (live + 31) & ~31;
    spmm_fixup_kernel<<<(unsigned)n_windows, wlive, 0, ctx->stream>>>(carry, carry_row, n_windows, Y, ldy, wlive, WIDTH);
    ctx->stats[0] += 2;
    return PB200_OK;
}

template <int LPT>
int launch_ldg(pb200_ctx* ctx, int64_t n_rows, const int64_t* indptr, const int32_t* indices, const float* values,
               const float* X, int64_t ldx, float* Y, int64_t ldy, int64_t nnz_begin, int64_t nnz_end, int live,
               int accumulate) {
    const int64_t n_blocks = std::max<int64_t>(1, ceil_div64(nnz_end - nnz_begin, CB));
    PB_REQUIRE(ctx, n_blocks < (int64_t)2147483647, "spmm: nnz too large for one launch");
    spmm_ldg_kernel<LPT><<<(unsigned)n_blocks, WARPS * 32, 0, ctx->stream>>>(n_rows, indptr, indices, values, X, ldx, Y, ldy,
                                                                           nnz_begin, n_blocks, live, accumulate);
    ctx->stats[0] += 1;
    return PB200_OK;
}

}  // namespace

// One (panel of a) CSR matrix times X: rows 0..n_rows-1 described by indptr[0..n_rows] (absolute nnz positions in
// [nnz_begin, nnz_end]); Y (+)= A X for the leading `ell` columns, Y written in whole groups of 32 columns.
int pb_spmm_panel(pb200_ctx* ctx, int64_t n_rows, const int64_t* indptr, const int32_t* indices, const float* values,
                  int64_t nnz_begin, int64_t nnz_end, const float* X, int64_t ldx, float* Y, int64_t ldy, int ell,
                  int accumulate) {
    PB_REQUIRE(ctx, ell > 0, "spmm: ell must be positive");
    PB_REQUIRE(ctx, n_rows >= 0 && nnz_end >= nnz_begin, "spmm: negative size");
    if (n_rows == 0) return PB200_OK;
    Scratch sc(ctx);
    // bulk copies need 16-byte aligned row segments that stay inside the row: ldx % 4 == 0, aligned base,
    // ldx >= ell rounded up to 4
    const bool staged = (ctx->spmm_kernel == 1 || ctx->spmm_kernel == 2) && (ldx % 4 == 0) &&
                        (reinterpret_cast<uintptr_t>(X) % 16 == 0) && ldx >= (ell + 3) / 4 * 4;
    const bool windowed = ctx->spmm_kernel == 3 || ctx->spmm_kernel == 4;
    // 128-bit gathers need 16-byte aligned row segments inside the row (Y too: it is written with 16-byte stores)
    const bool vec4 = ctx->spmm_kernel == 3 && (ldx % 4 == 0) && (ldy % 4 == 0) && (reinterpret_cast<uintptr_t>(X) % 16 == 0) &&
                      (reinterpret_cast<uintptr_t>(Y) % 16 == 0) && ldx >= (ell + 3) / 4 * 4 && ldx < ((int64_t)1 << 30);
    int done = 0;
    while (done < ell) {
        const int w = ell - done;                         // live columns left
        // lane occupancy: with 128-bit gathers a group of <= 64 columns keeps half a warp per nnz busy, 65..96 columns
        // only 24 of 32 lanes (those take the 32-bit kernel), 97..128 columns fill the warp again
        if (vec4 && w <= 64) {
            PB_TRY((launch_window4<false>(ctx, n_rows, indptr, indices, values, X + done, ldx, Y + done, ldy, nnz_begin, nnz_end,
                                          w, accumulate, sc)));
            done += 64;
            continue;
        }
        if (vec4 && w > 96) {
            PB_TRY((launch_window4<true>(ctx, n_rows, indptr, indices, values, X + done, ldx, Y + done, ldy, nnz_begin, nnz_end,
                                         std::min(w, 128), accumulate, sc)));
            done += 128;
            continue;
        }
        const float* x = X + done;
        float* y = Y + done;
        const int lpt = w > 96 ? 4 : w > 64 ? 3 : w > 32 ? 2 : 1;
        const int live = std::min(w, 32 * lpt);
#define PB_SPMM_CASE(L)                                                                                                   \
        if (windowed) PB_TRY((launch_window<L>(ctx, n_rows, indptr, indices, values, x, ldx, y, ldy, nnz_begin, nnz_end, live, \
                                               accumulate, sc)));                                                        \
        else if (staged) PB_TRY((launch_stage<L>(ctx, n_rows, indptr, indices, values, x, ldx, y, ldy, nnz_begin, nnz_end, live, \
                                            accumulate, sc)));                                                           \
        else PB_TRY((launch_ldg<L>(ctx, n_rows, indptr, indices, values, x, ldx, y, ldy, nnz_begin, nnz_end, live, accumulate)));
        switch (lpt) {
            case 4: PB_SPMM_CASE(4) break;
            case 3: PB_SPMM_CASE(3) break;
            case 2: PB_SPMM_CASE(2) break;
            default: PB_SPMM_CASE(1) break;
        }
#undef PB_SPMM_CASE
        done += 32 * lpt;
    }
    PB_CUDA(ctx, cudaGetLastError());
    return PB200_OK;
}

int pb_spmm_impl(pb200_ctx* ctx, int64_t n_rows, int64_t nnz, const int64_t* indptr,
                 const int32_t* indices, const float* values, const float* X, int64_t ldx,
                 float* Y, int64_t ldy, int ell) {
    return pb_spmm_panel(ctx, n_rows, indptr, indices, values, 0, nnz, X, ldx, Y, ldy, ell, 0);
}

// Panel-major matrix (pb200_csr_block_columns): panels run one after another, Y accumulates in panel order.
int pb_spmm_view(pb200_ctx* ctx, const pb200_csr_view* a, const float* X, int64_t ldx, float* Y, int64_t ldy, int ell) {
    PB_REQUIRE(ctx, a && a->indptr && a->n_panels >= 1, "spmm: bad matrix view");
    if (a->n_panels == 1) return pb_spmm_impl(ctx, a->n_rows, a->nnz, a->indptr, a->indices, a->values, X, ldx, Y, ldy, ell);
    PB_REQUIRE(ctx, a->panel_ptr_host != nullptr, "spmm: a panel-major matrix needs its host panel pointers");
    for (int p = 0; p < a->n_panels; ++p)
        PB_TRY(pb_spmm_panel(ctx, a->n_rows, a->indptr + (int64_t)p * a->n_rows, a->indices, a->values,
                             a->panel_ptr_host[p], a->panel_ptr_host[p + 1], X, ldx, Y, ldy, ell, p > 0));
    return PB200_OK;
}

extern "C" int pb200_spmm(pb200_ctx* ctx, int64_t n_rows, int64_t n_cols, int64_t nnz,
                          const int64_t* indptr, const int32_t* indices, const float* values,
                          const float* X, int64_t ldx, float* Y, int64_t ldy, int ell) {
    PB_ENTER(ctx);
    (void)n_cols;
    PB_REQUIRE(ctx, ldx >= ell && ldy >= (ell + 31) / 32 * 32, "spmm: need ldx >= ell and ldy >= ell rounded up to 32");
    return pb_spmm_impl(ctx, n_rows, nnz, indptr, indices, values, X, ldx, Y, ldy, ell);
}

extern "C" int pb200_spmm_csr(pb200_ctx* ctx, const pb200_csr_view* a, const float* X, int64_t ldx, float* Y,
                              int64_t ldy, int ell) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, a != nullptr, "spmm: null matrix view");
    PB_REQUIRE(ctx, ldx >= ell && ldy >= (ell + 31) / 32 * 32, "spmm: need ldx >= ell and ldy >= ell rounded up to 32");
    return pb_spmm_view(ctx, a, X, ldx, Y, ldy, ell);
}

// Fused scoring on the Hopper tensor cores (wgmma), sm_90a.
//
//   scores = E V^T  ->  seen-item mask  ->  per-user top-k          (score rows never reach HBM)
//
// replaces the dgemm of SVDModel.slice_recommendations (polara/recommender/models.py:857-861),
// downvote_seen_items (models.py:494-519) and get_topk_elements (models.py:522-564).
//
// Idea: the tensor cores only FILTER.  Operands are packed to bf16 (A = -E, B = V) together with
// three extra K-slots: a per-user threshold t_w (split hi+lo bf16, B holds 1.0 there) and a per-PAIR
// error margin (A: -(2^-7 + 2^-13) ||e_u||, B: ||v_j||, both rounded up), so the fp32 accumulator is
//     d = t_w - s~ - (2^-7 + 2^-13) ||e_u|| ||v_j||   with  s~ = bf16 dot product, |s~ - s| <= (2^-7 + 2^-16) ||e|| ||v||
// (bf16 unit round-off 2^-8 per operand; the 2^-13 and a 2^-16 |t_w| cut of the threshold pay for the fp32 accumulation).
// Items are swept in order of decreasing ||v_j|| (stable radix sort of the norms, CUB), which makes
// the running thresholds tight after the first tile.  The epilogue keeps ONLY THE SIGN BIT of each
// accumulator register: sign set  <=>  s~ + margin > t_w  <=>  "candidate".  t_w is a lower bound of the
// user's final k-th best exact score, so no true top-k item can be missed.
// Candidates (a few hundred per user out of 1e5 items) are then checked against the user's seen
// list and RESCORED EXACTLY in fp32 (the canonical fmaf chain of topk_common.cuh), which makes the
// result bit-identical to the exact SIMT kernel (topk_simt.cu).  As better candidates arrive the
// owner thread rewrites t_w inside the A operand in shared memory (generic-proxy store +
// fence.proxy.async), so later MMAs filter harder.
//
// Pipeline per CTA (persistent, one CTA per SM, 9 warps):
//   warp 8      producer : cp.async.bulk of pre-packed operand tiles (the A tile of the work item, then one 64-wide K
//                          slab of an item tile per ring stage), mbarrier complete_tx
//   warps 0-7   consumers: two warpgroups, each owns 64 users of the 128-user tile.  Per item tile a warpgroup issues
//                          wgmma.mma_async m64n128k16 (A and B from shared memory, 128-byte swizzle), collects the K slabs
//                          in 64 fp32 registers per thread, releases each ring stage as soon as its MMAs retired, then
//                          turns the signs into per-user candidate masks, stages them and rescores.
#include <cuda_bf16.h>
#include <cfloat>
#include <cstdlib>
#include <cub/device/device_radix_sort.cuh>

#include "topk_common.cuh"

namespace {

constexpr int BM = 128;          // users per tile (two warpgroups x 64)
constexpr int BN = 128;          // items per tile (wgmma N)
constexpr int NCONS = 256;       // consumer threads: two warpgroups
constexpr int NTHREADS = NCONS + 32;   // + the producer warp
constexpr int CAPS = 16;         // staged (chunk, mask) entries per consumer thread
constexpr int MAX_STAGES = 10;
constexpr uint32_t STAGE_BYTES = BN * 128;   // one ring stage: a 64-wide K slab (one 128-byte swizzle atom) of an item tile
constexpr int PROBE_ITEMS = 256; // largest-norm items scored exactly up front to seed the thresholds
constexpr int HEAD_TILES = 8;    // seen items among the first HEAD_TILES*BN sweep positions are masked by bitmap
constexpr int HEAD_WORDS = HEAD_TILES * BN / 32;
constexpr long long SPIN_LIMIT_CYCLES = 4000000000ll;

struct TcParams {
    const __nv_bfloat16* Ap;     // packed A tiles [user_tiles][BM x KP]
    const __nv_bfloat16* Bp;     // packed B tiles [item_tiles][BN x KP]
    const float* E; int64_t lde;
    const float* V; int64_t ldv;
    const int32_t* perm;         // [n] sweep position -> item id (norm-descending order)
    const float* t0;             // [m] seed lower bound of the k-th best score (or -inf)
    int64_t m, n;
    int r, KP, rs, k;
    int64_t user_tiles, item_tiles;
    int parts; int64_t tiles_per_part;
    int64_t tile_first;          // tiles [0, tile_first) hold the probe items, already scored exactly
    const int64_t* seen_indptr; const int32_t* seen_indices; int64_t seen_offset;
    pb200_cand* lists;           // [parts*2][m][k]
    int stages;
    uint32_t a_bytes, b_bytes;
    // early termination (null = sweep all, tile row i of user tile g is user g * BM + i): users sorted by the number of
    // item tiles they need, descending; tile row i of user tile g is user uperm[g * BM + i], which needs
    // need_sorted[g * BM + i] item tiles, so the first row of a tile needs the most
    const int32_t* uperm;        // [m]
    const int32_t* need_sorted;  // [m]
    const float* enorm;          // [m] ||e_u|| (inflated), by user id
    const float* vnorm_sorted;   // [n] ||v|| (inflated) by sweep position
    const uint32_t* headbits;    // [m][HEAD_WORDS] seen bitmap of the head of the sweep order (or null)
    unsigned long long* stats;   // device counters
    unsigned long long* hdbg;    // pinned host memory for timeout diagnostics (or null)
};

// The i-th work item of CTA c.  Work = (user tile, item part).  With early termination the user tiles cost between 1 and
// all item tiles: they are handed out longest first, each round of nc items in the opposite direction of the one before
// (CTA c gets ranks c, 2 nc - 1 - c, 2 nc + c, ...), which evens out the sums per CTA.
// Both roles of a CTA (producer, consumers) walk the same sequence through this function.
struct WorkItem { int64_t g; int part; };
__device__ __forceinline__ bool next_work(const TcParams& p, int64_t i, int64_t c, int64_t nc, int64_t n_groups, WorkItem& wk) {
    const bool rev = p.uperm != nullptr && (i & 1) && (i + 1) * nc <= n_groups;
    const int64_t w = i * nc + (rev ? nc - 1 - c : c);
    if (w >= n_groups) return false;
    wk.g = w / p.parts;                  // with early termination the user tiles come longest first already
    wk.part = (int)(w % p.parts);
    return true;
}

// ------------------------------------------------------------------ PTX wrappers --
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
__device__ __noinline__ void mbar_wait_slow(uint32_t bar, uint32_t parity, unsigned long long* stats, unsigned long long* g_hdbg) {
    uint32_t spins = 0;
    long long t_start = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0xFFFu) == 0) {        // never hang the GPU: after ~2 s record and abort the kernel
            long long now = clock64();
            if (t_start == 0) t_start = now;
            else if (now - t_start > SPIN_LIMIT_CYCLES) {
                if (stats) atomicExch(stats + 7, 0xDEAD0000ull | (bar & 0xFFFFu));
                if (g_hdbg && atomicCAS(g_hdbg, 0ull, 0xDEADull) == 0ull) {
                    g_hdbg[1] = bar; g_hdbg[2] = parity; g_hdbg[3] = threadIdx.x; g_hdbg[4] = blockIdx.x;
                    __threadfence_system();
                }
                asm volatile("trap;");
            }
        }
    }
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, unsigned long long* stats, unsigned long long* hdbg) {
    if (mbar_try_wait(bar, parity)) return;   // fast path
    mbar_wait_slow(bar, parity, stats, hdbg);
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving reads or writes of the accumulator registers across a wgmma fence / wait
__device__ __forceinline__ void wg_fence_acc(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 128] (+)= A[64 x 16] B[128 x 16]^T, both operands K-major bf16 in shared memory, fp32 accumulators in registers.
// Thread t of the warpgroup holds d[4 i + 2 a + b] = D[16 (t / 32) + (t % 32) / 4 + 8 a][8 i + 2 (t % 4) + b].
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, int accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// Operand tiles are K-major with the 128-byte swizzle: a tile of ROWS x KP bf16 is stored as
// ceil(KP/64) "atoms" of ROWS x 128 B; inside an atom row r sits at r*128 B and its eight 16-byte
// chunks are XOR-ed with (r % 8)  (Swizzle<3,4,3>); 8-row groups are 1024 B apart (SBO).  This is the
// layout wgmma reads with the SWIZZLE_128B descriptor; a K step of 16 inside an atom advances the start by 32 B.
__host__ __device__ __forceinline__ size_t tile_byte(int rows, int row, int k) {
    return (size_t)(k / 64) * ((size_t)rows * 128) + (size_t)(row / 8) * 1024 + (size_t)(row % 8) * 128 +
           (size_t)((((k % 64) / 8) ^ (row % 8)) * 16) + (size_t)(k % 8) * 2;
}
// wgmma shared-memory matrix descriptor: start address >> 4, LBO 16 B (unused with this swizzle), SBO = 1024 B,
// layout type 1 = SWIZZLE_128B (bits 62-63); atoms are 1024-byte aligned, so the base offset is 0
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// bf16 bit helpers (round toward -inf so that thresholds stay conservative)
__device__ __forceinline__ uint32_t bf16_floor_bits(float x) {
    uint32_t b = __float_as_uint(x);
    uint32_t hi = b >> 16;
    if ((b & 0xFFFFu) && (b >> 31)) hi += 1;     // negative: truncation rounds up -> step down
    return hi;
}
__device__ __forceinline__ uint32_t bf16_ceil_pos_bits(float x) {      // x >= 0, round up
    uint32_t b = __float_as_uint(x);
    return (b >> 16) + ((b & 0xFFFFu) ? 1u : 0u);
}
// pack threshold t (<= target) into {hi, lo} bf16 pair, hi + lo <= t
__device__ __forceinline__ uint32_t pack_threshold(float t) {
    if (!(t > -3.0e38f)) t = -3.0e38f;
    // explicit slack for the fp32 accumulation inside the tensor core (<= 67 additions, each 2^-24 relative to a partial sum
    // of size <= |t| + ||e|| ||v||): the |t| share is taken off the threshold here (2^-16 |t| >= 67 * 2^-24 |t|), the other share
    // is in the margin factor (pack_users_kernel).  FLT_MIN more puts the threshold strictly below a score of 0: where the
    // margin product is 0 (an item of norm 0, or ||e|| ||v|| 2^-7 under the accumulator's range) the accumulator would
    // otherwise sum to +0, and an item whose exact score ties a k-th score of 0 (and wins on its id) would not fire.  For
    // |t| >= 2^-86 the FLT_MIN is absorbed.
    t -= fabsf(t) * 1.52587890625e-5f + FLT_MIN;
    uint32_t hi = bf16_floor_bits(t);
    float hif = __uint_as_float(hi << 16);
    float rem = t - hif;                          // >= 0, exact
    uint32_t lo = bf16_floor_bits(rem);
    return (lo << 16) | (hi & 0xFFFFu);
}

// --------------------------------------------------------------- packing kernels --
__global__ void pack_items_kernel(const float* __restrict__ V, int64_t ldv, int64_t n, int r, int rs, int KP,
                                  int64_t item_tiles, const int32_t* __restrict__ perm,
                                  const float* __restrict__ vnorm_sorted, __nv_bfloat16* __restrict__ Bp) {
    const int chunks = (KP + 63) / 64 * 8;
    int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // one 16-byte chunk per thread
    int64_t total = item_tiles * BN * chunks;
    if (gid >= total) return;
    int64_t tile = gid / ((int64_t)BN * chunks);
    int rem = (int)(gid % ((int64_t)BN * chunks));
    int row = rem / chunks, ch = rem % chunks;
    int64_t pos = tile * BN + row;
    const int64_t item = pos < n ? (int64_t)__ldg(perm + pos) : -1;
    __align__(16) __nv_bfloat16 out[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        int kk = ch * 8 + j;
        float x = 0.f;
        if (item >= 0) {
            if (kk < r) x = __ldg(V + item * ldv + kk);
            else if (kk == rs || kk == rs + 1) x = 1.0f;
        }
        out[j] = __float2bfloat16_rn(x);
        if (item >= 0 && kk == rs + 2) out[j] = __ushort_as_bfloat16((unsigned short)bf16_ceil_pos_bits(__ldg(vnorm_sorted + pos)));
    }
    size_t byte = (size_t)tile * BN * chunks * 16 + tile_byte(BN, row, ch * 8);
    *reinterpret_cast<uint4*>(reinterpret_cast<unsigned char*>(Bp) + byte) = *reinterpret_cast<const uint4*>(out);
}

__global__ void pack_users_kernel(const float* __restrict__ E, int64_t lde, int64_t m, int r, int rs, int KP,
                                  int64_t user_tiles, const int32_t* __restrict__ uperm, const float* __restrict__ enorm,
                                  const float* __restrict__ t0, __nv_bfloat16* __restrict__ Ap) {
    const int chunks = (KP + 63) / 64 * 8;
    int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t total = user_tiles * BM * chunks;
    if (gid >= total) return;
    int64_t tile = gid / ((int64_t)BM * chunks);
    int rem = (int)(gid % ((int64_t)BM * chunks));
    int row = rem / chunks, ch = rem % chunks;
    const int64_t tr = tile * BM + row;                               // tile row; padding rows (tr >= m) stay zero
    const int64_t u = (tr < m && uperm) ? (int64_t)__ldg(uperm + tr) : tr;
    __align__(16) __nv_bfloat16 out[8];
    uint32_t thr = 0;
    if (ch == rs / 8) {
        if (u < m) {
            thr = pack_threshold(t0[u]);
        } else {
            thr = 0x00007F7Fu;                                            // +3.39e38: padding rows never fire
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        int kk = ch * 8 + j;
        float x = 0.f;
        if (u < m && kk < r) x = -__ldg(E + u * lde + kk);
        out[j] = __float2bfloat16_rn(x);
        if (kk == rs) out[j] = __ushort_as_bfloat16((unsigned short)(thr & 0xFFFFu));
        if (kk == rs + 1) out[j] = __ushort_as_bfloat16((unsigned short)(thr >> 16));
        // per-pair margin slot: -((2^-7 + 2^-13) ||e_u||) rounded away from zero.  bf16 rounding: unit round-off u = 2^-8 per
        // operand, so |s~ - s| <= (2u + u^2) sum|e_i v_i| <= (2^-7 + 2^-16) ||e|| ||v||; the extra 2^-13 - 2^-16 covers the
        // tensor core's fp32 accumulation of the ||e|| ||v||-sized terms (67 * 2^-24 < 2^-17) with room to spare
        if (kk == rs + 2 && u < m)
            out[j] = __ushort_as_bfloat16((unsigned short)(0x8000u | bf16_ceil_pos_bits(0.0079345703125f * enorm[u] + 1e-30f)));
    }
    size_t byte = (size_t)tile * BM * chunks * 16 + tile_byte(BM, row, ch * 8);
    *reinterpret_cast<uint4*>(reinterpret_cast<unsigned char*>(Ap) + byte) = *reinterpret_cast<const uint4*>(out);
}

// row norms (one warp per row); optional max over rows (positive floats order like ints)
__global__ void row_norm_kernel(const float* __restrict__ X, int64_t ld, int64_t rows, int r, float* __restrict__ norms,
                                float* __restrict__ max_out) {
    int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (w >= rows) return;
    float s = 0.f;
    for (int t = lane; t < r; t += 32) { float x = __ldg(X + w * ld + t); s = fmaf(x, x, s); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    s = sqrtf(s) * 1.0001f;                    // tiny inflation covers the rounding of the norm itself
    if (lane == 0) {
        if (norms) norms[w] = s;
        if (max_out) atomicMax(reinterpret_cast<int*>(max_out), __float_as_int(s));
    }
}

__global__ void iota_i32_kernel(int32_t* __restrict__ x, int64_t n) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] = (int32_t)i;
}

__global__ void invert_perm_kernel(const int32_t* __restrict__ perm, int64_t n, int32_t* __restrict__ inv) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) inv[perm[i]] = (int32_t)i;
}

// bit (31 - pos%32) of word pos/32 of user u is set when the item at sweep position pos (< HEAD_TILES*256)
// is in u's seen list; one warp per user
// bit (item % 32) of word item / 32 is set when the item sits inside the head of the sweep order
__global__ void head_items_kernel(const int32_t* __restrict__ perm, int64_t n_head, uint32_t* __restrict__ in_head) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_head) { const int32_t item = perm[i]; atomicOr(in_head + (item >> 5), 1u << (item & 31)); }
}

__global__ void __launch_bounds__(256)
head_bitmap_kernel(const int64_t* __restrict__ seen_indptr, const int32_t* __restrict__ seen_indices,
                   int64_t seen_offset, const int32_t* __restrict__ inv_perm, const uint32_t* __restrict__ in_head,
                   int64_t m, int64_t n, uint32_t* __restrict__ bits) {
    // one warp per user: the HEAD_WORDS (= 32) words of the row are assembled in shared memory and written once
    static_assert(HEAD_WORDS == 32, "one bitmap word per lane");
    __shared__ uint32_t sw[8][HEAD_WORDS];
    const int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (u >= m) return;
    sw[warp][lane] = 0u;
    __syncwarp();
    for (int64_t p = seen_indptr[u] + lane; p < seen_indptr[u + 1]; p += 32) {
        int64_t item = (int64_t)__ldg(seen_indices + p) - seen_offset;
        if (item < 0 || item >= n) continue;
        // the membership words (n / 8 bytes) stay in L1; the position table (4 n bytes) is read for head items only
        if (!((__ldg(in_head + (item >> 5)) >> (item & 31)) & 1u)) continue;
        int pos = __ldg(inv_perm + item);
        atomicOr(&sw[warp][pos >> 5], 0x80000000u >> (pos & 31));
    }
    __syncwarp();
    bits[u * HEAD_WORDS + lane] = sw[warp][lane];
}

// Early termination of the norm-ordered sweep (exact).  Items are visited by decreasing ||v||; by Cauchy-Schwarz the
// canonical fp32 score of (u, item at position p) is at most enorm[u] * vnorm_sorted[p] (both norms are inflated by 1.0001,
// which also covers the rounding of the fp32 fmaf chain, <= r * 2^-24 relative).  Any lower bound t of the user's final
// k-th best score (t0 from the probe, later the k-th scores of the sweep's own lists) makes every position with
// enorm * vnorm < t (strictly: a tie could still win on the item id) irrelevant for u, and all later ones too.
// Returns the first item tile in [lo, hi] whose first position has a bound below t -- the user needs no tile from there
// on -- or hi (t not positive and finite: no cut).  hi <= item tiles, so every probed position exists.
__device__ __forceinline__ int first_cut_tile(float en, float t, const float* __restrict__ vnorm_sorted, int lo, int hi) {
    if (!(t > 0.f && t < CUDART_INF_F)) return hi;
    while (lo < hi) {                                     // bounds are non-increasing along the sweep
        const int mid = (lo + hi) >> 1;
        if (en * __ldg(vnorm_sorted + (int64_t)mid * BN) < t) hi = mid; else lo = mid + 1;
    }
    return lo;
}

// need[u] = item tiles user u needs under its bound t0[u]; used when the bounds changed after the probe (bound hook)
__global__ void user_need_kernel(const float* __restrict__ enorm, const float* __restrict__ t0,
                                 const float* __restrict__ vnorm_sorted, int64_t m, int item_tiles, int32_t* __restrict__ need) {
    const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (u < m) need[u] = first_cut_tile(__ldg(enorm + u), __ldg(t0 + u), vnorm_sorted, 0, item_tiles);
}

// Exact fp32 scores of 64 users x the PROBE_ITEMS largest-norm items; t0[u] = k-th largest unseen
// score (a valid lower bound of the user's final k-th best score), -inf if fewer than k are unseen.
// The probe reads every row of E anyway, so it also emits enorm[u] (the row norm, inflated like row_norm_kernel's) and,
// when need is not null, need[u] = first_cut_tile under t0[u].
constexpr int PTU = 64, PTI = 128, PKS = 32;
constexpr int PNU = 2;                          // users a warp selects for at the same time (independent latency chains)
template <int PI>
struct ProbeSmem {
    float es[PKS][PTU + 4];
    float vs[PKS][PTI + 4];
    float sc[PTU][PI + 4];                      // row stride = 4 mod 32 words: 16-byte row stores and lane-strided reads, no conflicts
    unsigned long long cand[8][PNU][32];        // per warp and user in flight: the keys that can still be among the k best
    float t0s[PTU];
};

// order-preserving 32-bit image of a float (larger float <=> larger unsigned) and its inverse
__device__ __forceinline__ uint32_t ord_of(float x) {
    const uint32_t b = __float_as_uint(x);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord_to_float(uint32_t o) {
    return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o);
}

// Reference selection (any k, any number of ties): every lane sorts its keys once, then k rounds pop the warp-wide best
// head.  key = ord(score) << 32 | ~id, 0 = masked / absent; a larger key ranks earlier under (score desc, id asc).
template <int PL>
__device__ __noinline__ void probe_select_rounds(unsigned long long (&key)[PL], int lane, int k,
                                                 pb200_cand* __restrict__ out, float* __restrict__ t0_u) {
    static_assert(PL == 8, "the sorting network below is for 8 keys per lane");
#define PB_CAS(A, B) { const unsigned long long x_ = key[A], y_ = key[B]; const bool g_ = x_ > y_; key[A] = g_ ? x_ : y_; key[B] = g_ ? y_ : x_; }
    PB_CAS(0, 1) PB_CAS(2, 3) PB_CAS(4, 5) PB_CAS(6, 7)
    PB_CAS(0, 2) PB_CAS(1, 3) PB_CAS(4, 6) PB_CAS(5, 7)
    PB_CAS(1, 2) PB_CAS(5, 6)
    PB_CAS(0, 4) PB_CAS(1, 5) PB_CAS(2, 6) PB_CAS(3, 7)
    PB_CAS(2, 4) PB_CAS(3, 5)
    PB_CAS(1, 2) PB_CAS(3, 4) PB_CAS(5, 6)
#undef PB_CAS
    float kth = -CUDART_INF_F;
    int produced = 0;
    pb200_cand mine; mine.score = -CUDART_INF_F; mine.id = -1;
    for (; produced < k; ++produced) {
        const uint32_t hh = (uint32_t)(key[0] >> 32), hl = (uint32_t)key[0];
        const uint32_t wh = __reduce_max_sync(0xffffffffu, hh);
        if (wh == 0u) break;                                             // fewer than k unseen probe items
        const uint32_t wl = __reduce_max_sync(0xffffffffu, hh == wh ? hl : 0u);   // ~id >= 2^31 > 0 for every real key
        if (hh == wh && hl == wl) {                                      // ids are unique: exactly one lane pops
#pragma unroll
            for (int j = 0; j + 1 < PL; ++j) key[j] = key[j + 1];
            key[PL - 1] = 0ull;
        }
        const float ws = ord_to_float(wh);
        if (lane == (produced & 31)) { mine.score = ws; mine.id = (int)(0xFFFFFFFFu - wl); }
        if ((produced & 31) == 31) out[(produced - 31) + lane] = mine;
        kth = ws;
    }
    if (lane < (produced & 31)) out[(produced & ~31) + lane] = mine;
    for (int j = produced + lane; j < k; j += 32) { pb200_cand c; c.score = -CUDART_INF_F; c.id = -1; out[j] = c; }
    if (lane == 0) *t0_u = produced == k ? kth : -CUDART_INF_F;
}

template <int PI>
__global__ void __launch_bounds__(256)
probe_kernel(const float* __restrict__ E, int64_t lde, const float* __restrict__ V, int64_t ldv,
             const int32_t* __restrict__ perm, int64_t m, int64_t n_probe, int r, int k,
             const uint32_t* __restrict__ headbits, float* __restrict__ t0, pb200_cand* __restrict__ out_list,
             float* __restrict__ enorm, const float* __restrict__ vnorm_sorted, int item_tiles, int32_t* __restrict__ need) {
    extern __shared__ __align__(16) unsigned char praw[];
    ProbeSmem<PI>& sm = *reinterpret_cast<ProbeSmem<PI>*>(praw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, tx = tid & 15, ty = tid >> 4;
    const int64_t u0 = (int64_t)blockIdx.x * PTU;
    // 128-bit tile loads when every row segment is 16-byte aligned (the engine's padded factors always are)
    const bool vec = ((lde | ldv) & 3) == 0 && ((reinterpret_cast<uintptr_t>(E) | reinterpret_cast<uintptr_t>(V)) & 15) == 0;
    const int n_ktiles = (r + PKS - 1) / PKS, n_tiles = (PI / PTI) * n_ktiles;
    // vector path: a thread owns one user row (tid & 63) and one item row (tid & 127) of the tile and a fixed set of K
    // quads; the next tile's quads are fetched into registers while the current tile is multiplied
    const int64_t eu = u0 + (tid & (PTU - 1));
    const float* erow = eu < m ? E + eu * lde : nullptr;
    const float* vrow = nullptr;
    float4 pe[2], pv[4];
    auto fetch = [&](int tile) {
        const int i0 = (tile / n_ktiles) * PTI, k0 = (tile % n_ktiles) * PKS;
        if (tile % n_ktiles == 0) {
            const int64_t vpos = i0 + (tid & (PTI - 1));
            vrow = vpos < n_probe ? V + (int64_t)__ldg(perm + vpos) * ldv : nullptr;
        }
#pragma unroll
        for (int it = 0; it < 2; ++it) {
            const int kq = k0 + 4 * ((tid >> 6) + 4 * it);
            pe[it] = (erow && kq < r) ? __ldg(reinterpret_cast<const float4*>(erow + kq)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int it = 0; it < 4; ++it) {
            const int kq = k0 + 4 * ((tid >> 7) + 2 * it);
            pv[it] = (vrow && kq < r) ? __ldg(reinterpret_cast<const float4*>(vrow + kq)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    auto stash = [&](int tile) {              // registers -> transposed shared-memory tiles (one lane per row: no conflicts)
        const int k0 = (tile % n_ktiles) * PKS;
#pragma unroll
        for (int it = 0; it < 2; ++it) {
            const int q = (tid >> 6) + 4 * it, kq = k0 + 4 * q, row = tid & (PTU - 1);
            sm.es[4 * q + 0][row] = pe[it].x;
            sm.es[4 * q + 1][row] = kq + 1 < r ? pe[it].y : 0.f;      // K quads at or beyond r are never multiplied; inside
            sm.es[4 * q + 2][row] = kq + 2 < r ? pe[it].z : 0.f;      // the last quad the padding of the row is cut here
            sm.es[4 * q + 3][row] = kq + 3 < r ? pe[it].w : 0.f;
        }
#pragma unroll
        for (int it = 0; it < 4; ++it) {
            const int q = (tid >> 7) + 2 * it, kq = k0 + 4 * q, row = tid & (PTI - 1);
            sm.vs[4 * q + 0][row] = pv[it].x;
            sm.vs[4 * q + 1][row] = kq + 1 < r ? pv[it].y : 0.f;
            sm.vs[4 * q + 2][row] = kq + 2 < r ? pv[it].z : 0.f;
            sm.vs[4 * q + 3][row] = kq + 3 < r ? pv[it].w : 0.f;
        }
    };
    if (vec) fetch(0);
    float acc[4][8];
    float en2 = 0.f;                          // threads 0..PTU-1: squared norm of user u0 + tid
    for (int tile = 0; tile < n_tiles; ++tile) {
        const int i0 = (tile / n_ktiles) * PTI, k0 = (tile % n_ktiles) * PKS;
        if (k0 == 0) {
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 8; ++b) acc[a][b] = 0.f;
        }
        if (vec) {
            stash(tile);
        } else {
#pragma unroll
            for (int it = 0; it < 8; ++it) {
                int e = tid + it * 256, row = e >> 5, kk = e & 31;
                int64_t u = u0 + row;
                sm.es[kk][row] = (u < m && k0 + kk < r) ? __ldg(E + u * lde + k0 + kk) : 0.f;
            }
#pragma unroll
            for (int it = 0; it < 16; ++it) {
                int e = tid + it * 256, row = e >> 5, kk = e & 31;
                int64_t pos = i0 + row;
                sm.vs[kk][row] = (pos < n_probe && k0 + kk < r) ? __ldg(V + (int64_t)__ldg(perm + pos) * ldv + k0 + kk) : 0.f;
            }
        }
        __syncthreads();
        if (vec && tile + 1 < n_tiles) fetch(tile + 1);
        const int kmax = min(PKS, r - k0);
        if (i0 == 0 && tid < PTU)             // the first item block walks all K tiles of E once
            for (int kk = 0; kk < kmax; ++kk) en2 = fmaf(sm.es[kk][tid], sm.es[kk][tid], en2);
        // thread (tx, ty): users 4 ty .. 4 ty + 3, items 4 tx .. 4 tx + 3 and 64 + 4 tx .. 64 + 4 tx + 3 of the tile, so that
        // the 16 lanes of a half-warp read one contiguous 256-byte run per load
        for (int kk = 0; kk < kmax; ++kk) {
            float4 e4 = *reinterpret_cast<const float4*>(&sm.es[kk][ty * 4]);
            float4 v0 = *reinterpret_cast<const float4*>(&sm.vs[kk][tx * 4]);
            float4 v1 = *reinterpret_cast<const float4*>(&sm.vs[kk][64 + tx * 4]);
            float a[4] = {e4.x, e4.y, e4.z, e4.w};
            float b[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (k0 + PKS >= r) {                   // last K tile of this item block: scores to shared memory (16-byte stores)
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int hseg = 0; hseg < 2; ++hseg) {
                    const int pos = i0 + 64 * hseg + tx * 4;
                    float4 x;
                    x.x = pos + 0 < n_probe ? acc[i][4 * hseg + 0] : -CUDART_INF_F;
                    x.y = pos + 1 < n_probe ? acc[i][4 * hseg + 1] : -CUDART_INF_F;
                    x.z = pos + 2 < n_probe ? acc[i][4 * hseg + 2] : -CUDART_INF_F;
                    x.w = pos + 3 < n_probe ? acc[i][4 * hseg + 3] : -CUDART_INF_F;
                    *reinterpret_cast<float4*>(&sm.sc[ty * 4 + i][pos]) = x;
                }
        }
        __syncthreads();
    }
    // Exact top-k of the probe set per user under the list order (score desc, id asc); one warp per user, lane owns the
    // positions lane + 32 j.  Fast path (k <= 32): the k-th largest of the 32 lane maxima is a threshold tau with at least k
    // keys at or above it; those few keys (k plus the handful of second-best entries of the winning lanes) are compacted
    // into shared memory, every lane ranks one of them by counting the larger ones, and rank i goes to slot i of the list.
    // More than 32 keys at or above tau (ties: e.g. an all-zero embedding) or k > 32 take the reference selection.
    // A warp works on PNU users at a time: their chains of dependent steps (bitmap load, k reductions, id load) interleave.
    constexpr int PL = PI / 32;                                                // keys per lane
    const uint32_t lt_mask = (1u << lane) - 1u;
    for (int ul = warp; ul < PTU; ul += 8 * PNU) {
        int64_t u[PNU];
        bool act[PNU];
        uint32_t seen_w[PNU], ord[PNU][PL], lmax[PNU], tau[PNU];
        int count[PNU] = {};
#pragma unroll
        for (int a = 0; a < PNU; ++a) {
            u[a] = u0 + ul + 8 * a;
            act[a] = ul + 8 * a < PTU && u[a] < m;                             // warp-uniform
            seen_w[a] = 0u;                                                    // lane j < PL: word j covers positions 32j..32j+31
            if (act[a] && headbits && lane < PL) seen_w[a] = __ldg(headbits + u[a] * HEAD_WORDS + lane);
        }
#pragma unroll
        for (int a = 0; a < PNU; ++a) {
            lmax[a] = 0u;
#pragma unroll
            for (int j = 0; j < PL; ++j) {
                const int pos = lane + 32 * j;
                const uint32_t w = __shfl_sync(0xffffffffu, seen_w[a], j);
                const bool ok = act[a] && pos < n_probe && !(w & (0x80000000u >> lane));
                // + 0.f turns -0 into +0: the two zeros tie and the id decides, as in cand_before (ord_of alone puts -0
                // below +0); the sign of a zero score is restored after the selection
                ord[a][j] = ok ? ord_of(sm.sc[act[a] ? ul + 8 * a : 0][pos] + 0.f) : 0u;
                lmax[a] = max(lmax[a], ord[a][j]);
            }
        }
        const bool small_k = k <= 32;
        if (small_k) {
            uint32_t rest[PNU], w[PNU];
#pragma unroll
            for (int a = 0; a < PNU; ++a) { rest[a] = lmax[a]; w[a] = 0u; }
            for (int i = 0; i < k; ++i) {                                      // lanes that tie leave together: tau can only
#pragma unroll
                for (int a = 0; a < PNU; ++a) {                                // come out lower, never too high
                    w[a] = __reduce_max_sync(0xffffffffu, rest[a]);
                    if (rest[a] == w[a]) rest[a] = 0u;
                }
            }
#pragma unroll
            for (int a = 0; a < PNU; ++a) tau[a] = w[a] == 0u ? 1u : w[a];     // fewer than k lanes hold a key: take every key
#pragma unroll
            for (int a = 0; a < PNU; ++a) count[a] = 0;
#pragma unroll
            for (int j = 0; j < PL; ++j)
#pragma unroll
                for (int a = 0; a < PNU; ++a) {
                    const bool in = ord[a][j] >= tau[a];
                    const uint32_t b = __ballot_sync(0xffffffffu, in);
                    const int slot = count[a] + __popc(b & lt_mask);
                    if (in && slot < 32) sm.cand[warp][a][slot] = ((unsigned long long)ord[a][j] << 32) | (uint32_t)(lane + 32 * j);
                    count[a] += __popc(b);
                }
        }
        bool fast[PNU];
#pragma unroll
        for (int a = 0; a < PNU; ++a) fast[a] = act[a] && small_k && count[a] <= 32;
        __syncwarp();
        unsigned long long mine[PNU];
        uint32_t mpos[PNU];                                                    // probe position of this lane's key
#pragma unroll
        for (int a = 0; a < PNU; ++a) {
            mine[a] = 0ull;
            mpos[a] = 0u;
            if (fast[a] && lane < count[a]) {
                const unsigned long long c = sm.cand[warp][a][lane];
                mpos[a] = (uint32_t)c;
                const uint32_t id = (uint32_t)__ldg(perm + (uint32_t)c);
                mine[a] = (c & 0xFFFFFFFF00000000ull) | (unsigned long long)(0xFFFFFFFFu - id);
            }
        }
        __syncwarp();
#pragma unroll
        for (int a = 0; a < PNU; ++a) if (fast[a]) sm.cand[warp][a][lane] = mine[a];
        __syncwarp();
#pragma unroll
        for (int a = 0; a < PNU; ++a) {
            if (!fast[a]) continue;
            pb200_cand* out = out_list + u[a] * k;
            int rank = 0;
            for (int t = 0; t < count[a]; ++t) rank += sm.cand[warp][a][t] > mine[a] ? 1 : 0;
            if (lane < count[a] && rank < k) {
                pb200_cand c; c.score = ord_to_float((uint32_t)(mine[a] >> 32)); c.id = (int)(0xFFFFFFFFu - (uint32_t)mine[a]);
                if (c.score == 0.f) c.score = sm.sc[ul + 8 * a][mpos[a]];  // the key ranked -0 as +0: the canonical sign
                out[rank] = c;
                if (rank == k - 1) sm.t0s[ul + 8 * a] = c.score;
            }
            if (count[a] < k) {
                if (lane >= count[a] && lane < k) { pb200_cand c; c.score = -CUDART_INF_F; c.id = -1; out[lane] = c; }
                if (lane == 0) sm.t0s[ul + 8 * a] = -CUDART_INF_F;
            }
        }
        __syncwarp();
#pragma unroll
        for (int a = 0; a < PNU; ++a) {
            if (!act[a] || fast[a]) continue;
            unsigned long long key[PL];
#pragma unroll
            for (int j = 0; j < PL; ++j) {
                const uint32_t id = ord[a][j] ? (uint32_t)__ldg(perm + lane + 32 * j) : 0u;
                key[j] = ord[a][j] ? (((unsigned long long)ord[a][j] << 32) | (unsigned long long)(0xFFFFFFFFu - id)) : 0ull;
            }
            probe_select_rounds<PL>(key, lane, k, out_list + u[a] * k, &sm.t0s[ul + 8 * a]);
        }
        // the reference selection's keys ranked a -0 score as +0 and carry no position: a zero score is recomputed, so that
        // its sign is the canonical one (the fast path restored it from the score tile above)
        __syncwarp();
#pragma unroll
        for (int a = 0; a < PNU; ++a) {
            if (!act[a] || fast[a]) continue;
            pb200_cand* out = out_list + u[a] * k;
            for (int j = lane; j < k; j += 32) {
                const pb200_cand c = out[j];
                if (c.id >= 0 && c.score == 0.f) out[j].score = exact_score(E + u[a] * lde, V + (int64_t)c.id * ldv, r);
            }
        }
    }
    __syncthreads();
    if (tid < PTU && u0 + tid < m) {
        const int64_t uu = u0 + tid;
        const float t = sm.t0s[tid], en = sqrtf(en2) * 1.0001f;      // tiny inflation covers the rounding of the norm itself
        t0[uu] = t;
        enorm[uu] = en;
        if (need) need[uu] = first_cut_tile(en, t, vnorm_sorted, 0, item_tiles);
    }
}

// ------------------------------------------------------------------ main kernel ---
// canonical fp32 score (fmaf chain, ascending k); 128-bit loads are issued 8 at a time so that the L2 latency is paid
// once per batch instead of once per element
__device__ __forceinline__ float exact_score_vec(const float* __restrict__ erow, const float* __restrict__ vrow, int r, bool vec_ok) {
    if (!vec_ok) return exact_score(erow, vrow, r);
    const int r4 = r / 4;
    const float4* e4 = reinterpret_cast<const float4*>(erow);
    const float4* v4 = reinterpret_cast<const float4*>(vrow);
    float s = 0.f;
    int t = 0;
    for (; t + 8 <= r4; t += 8) {
        float4 a[8], b[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) { a[i] = __ldg(e4 + t + i); b[i] = __ldg(v4 + t + i); }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            s = fmaf(a[i].x, b[i].x, s); s = fmaf(a[i].y, b[i].y, s);
            s = fmaf(a[i].z, b[i].z, s); s = fmaf(a[i].w, b[i].w, s);
        }
    }
    for (; t + 4 <= r4; t += 4) {
        float4 a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { a[i] = __ldg(e4 + t + i); b[i] = __ldg(v4 + t + i); }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            s = fmaf(a[i].x, b[i].x, s); s = fmaf(a[i].y, b[i].y, s);
            s = fmaf(a[i].z, b[i].z, s); s = fmaf(a[i].w, b[i].w, s);
        }
    }
    for (; t < r4; ++t) {
        float4 a = __ldg(e4 + t), b = __ldg(v4 + t);
        s = fmaf(a.x, b.x, s); s = fmaf(a.y, b.y, s); s = fmaf(a.z, b.z, s); s = fmaf(a.w, b.w, s);
    }
    for (int tt = r4 * 4; tt < r; ++tt) s = fmaf(__ldg(erow + tt), __ldg(vrow + tt), s);
    return s;
}

struct ListState {
    pb200_cand* list;   // k slots in global memory, sorted
    int cnt;
    float kth;          // score of slot k-1 once full, else -inf
};

__device__ __forceinline__ void list_insert(ListState& ls, int k, float s, int id) {
    if (ls.cnt == k) {
        pb200_cand last = ls.list[k - 1];
        if (!cand_before(s, id, last.score, last.id)) return;
    }
    int i = ls.cnt < k ? ls.cnt : k - 1;
    while (i > 0) {
        pb200_cand p = ls.list[i - 1];
        if (!cand_before(s, id, p.score, p.id)) break;
        ls.list[i] = p;
        --i;
    }
    pb200_cand c; c.score = s; c.id = id;
    ls.list[i] = c;
    if (ls.cnt < k) ls.cnt++;
    if (ls.cnt == k) ls.kth = ls.list[k - 1].score;
}

// One row's staged survivors, worked on by the whole warp: lane c takes column c of every staged 32-column chunk (sweep
// position -> item -> seen test -> exact score), the passing ones enter the row's list through warp_list_insert.  For rows
// whose threshold filters nothing (a user whose history covers the head of the sweep order): 16 staged chunks are up to 512
// survivors, which the owning thread alone would work off one after the other; the warp takes 32 at a time, 16 steps.  Same results: the list is the set of the k best under a strict
// order, whoever inserts.  Returns the number of exact scores computed by this lane.
constexpr int COOP_MIN = 64;     // survivors in one flush from which a row is handed to the whole warp
struct CoopArgs {                // the few kernel parameters the cooperative flush reads (passed by value: no local copy of TcParams)
    const float* V; int64_t ldv; const int32_t* perm; const int32_t* seen_indices; int64_t seen_offset; int64_t n; int r, k;
};
__device__ __noinline__ int coop_flush_row(const CoopArgs p, const float* __restrict__ erow, const uint2* __restrict__ stage_row,
                                           int n_entries, int64_t t_lo, int64_t sb, int64_t se, bool head_masked,
                                           pb200_cand* __restrict__ list, float t_row, bool vec_ok, int lane, int& cnt, float& kth) {
    int n_scored = 0;
    for (int e = 0; e < n_entries; ++e) {
        const uint2 ent = stage_row[e * 256];
        const int64_t pos = (int64_t)(t_lo + (ent.x >> 2)) * BN + (ent.x & 3) * 32 + lane;
        bool ok = ((ent.y << lane) & 0x80000000u) != 0u && pos < p.n;             // column c <-> bit 31-c
        int item = -1;
        float s = 0.f;
        if (ok) {
            item = __ldg(p.perm + pos);
            if (sb < se && (!head_masked || pos >= HEAD_TILES * BN) &&
                seen_lookup(p.seen_indices, sb, se, (int)(item + p.seen_offset))) ok = false;
        }
        if (ok) {
            s = exact_score_vec(erow, p.V + (int64_t)item * p.ldv, p.r, vec_ok);
            ++n_scored;
            ok = !(s < t_row);
        }
        uint32_t pass = __ballot_sync(0xffffffffu, ok);
        while (pass) {
            const int l = __ffs(pass) - 1;
            pass &= pass - 1;
            const float sl = __shfl_sync(0xffffffffu, s, l);
            const int il = __shfl_sync(0xffffffffu, item, l);
            if (sl < t_row) continue;                                             // the bound may have risen since the ballot
            cnt = warp_list_insert(list, p.k, cnt, sl, il, lane);
            if (cnt == p.k) { kth = list[p.k - 1].score; t_row = fmaxf(t_row, kth); }
        }
    }
    return n_scored;
}

__global__ void __launch_bounds__(NTHREADS, 1)
score_topk_tc_kernel(const TcParams p) {
    extern __shared__ __align__(1024) unsigned char smem[];
    // ---- carve shared memory -------------------------------------------------------
    unsigned char* sA = smem + ((1024u - (smem_u32(smem) & 1023u)) & 1023u);     // swizzle atoms need 1024 B alignment
    unsigned char* sB = sA + p.a_bytes;
    uint2* sStage = reinterpret_cast<uint2*>(sB + (size_t)p.stages * STAGE_BYTES);          // [CAPS][256]
    volatile uint2* sThr = reinterpret_cast<volatile uint2*>(sStage + CAPS * 256);          // [2][128] {work tag, k-th score}
    uint64_t* bars = reinterpret_cast<uint64_t*>(const_cast<uint2*>(sThr) + 256);
    // barrier layout: full[MAX_STAGES], empty[MAX_STAGES], a_full, a_empty
    const uint32_t bar_full = smem_u32(bars), bar_empty = smem_u32(bars + MAX_STAGES);
    const uint32_t bar_afull = smem_u32(bars + 2 * MAX_STAGES), bar_aempty = smem_u32(bars + 2 * MAX_STAGES + 1);
    // flush generation of this CTA: a warp that has to work off its staged survivors bumps it, the other seven follow at
    // their next tile.  The warps of a warpgroup meet at every wgmma, so they may as well rescore at the same time.
    volatile uint32_t* flush_gen = reinterpret_cast<volatile uint32_t*>(bars + 2 * MAX_STAGES + 2);
    // live cut (early termination only): consumer warp w publishes {work tag, item tile from which none of its rows needs
    // anything} in sCut[w]; the producer stops the work item's sweep once it reaches the largest of the eight.  It tells
    // the consumers by one extra stage that carries no data and has sStop[stage] set.
    volatile unsigned long long* sCut = reinterpret_cast<volatile unsigned long long*>(bars + 2 * MAX_STAGES + 4);   // [8]
    volatile uint32_t* sStop = reinterpret_cast<volatile uint32_t*>(bars + 2 * MAX_STAGES + 4 + NCONS / 32);         // [MAX_STAGES]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // tags of a previous launch may still sit in this shared memory: a stale entry that happened to carry this launch's
    // work tag would be taken for a valid lower bound of another user's k-th score (or for another tile's cut)
    if (tid < 256) { const_cast<uint2*>(sThr)[tid] = make_uint2(0u, 0u); }
    if (tid < NCONS / 32) sCut[tid] = 0ull;
    if (tid < MAX_STAGES) sStop[tid] = 0u;
    if (tid == 0) {
        *flush_gen = 0u;
        for (int s = 0; s < p.stages; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, NCONS / 32); }
        mbar_init(bar_afull, 1);
        mbar_init(bar_aempty, NCONS / 32);
        fence_barrier_init();
        if (p.hdbg && blockIdx.x == 0) p.hdbg[5] = bar_full;     // lets a timeout report be decoded: (bar - base) / 8 = barrier index
    }
    __syncthreads();

    const int64_t n_groups = p.user_tiles * p.parts;
    const int64_t n_ctas = gridDim.x, cta = blockIdx.x;
    WorkItem wk;
    const uint32_t S = (uint32_t)p.stages;
    const int KA = (p.KP + 63) / 64;                   // K slabs per item tile

    if (warp == NCONS / 32) {
        // ============================ producer ======================================
        if (lane == 0) {
            uint32_t stage = 0, phase = 0, awork = 0;
            for (int64_t wi = 0; next_work(p, wi, cta, n_ctas, n_groups, wk); ++wi, ++awork) {
                const int64_t t_lo = min(p.item_tiles, p.tile_first + (int64_t)wk.part * p.tiles_per_part);
                int64_t t_hi = min(p.item_tiles, p.tile_first + (int64_t)(wk.part + 1) * p.tiles_per_part);
                if (p.need_sorted) t_hi = min(t_hi, max(t_lo, (int64_t)__ldg(p.need_sorted + wk.g * BM)));
                mbar_wait(bar_aempty, (awork & 1) ^ 1, p.stats, p.hdbg);
                mbar_arrive_expect_tx(bar_afull, p.a_bytes);
                bulk_g2s(smem_u32(sA), reinterpret_cast<const unsigned char*>(p.Ap) + (size_t)wk.g * p.a_bytes, p.a_bytes, bar_afull);
                for (int64_t t = t_lo; t < t_hi; ++t) {
                    if (p.need_sorted) {
                        // the consumers of this work item only publish after the A tile landed, so every entry still
                        // carries an older tag until all eight warps have spoken
                        bool all = true;
                        int64_t live_cut = 0;
#pragma unroll
                        for (int w = 0; w < NCONS / 32; ++w) {
                            const unsigned long long e = sCut[w];
                            all = all && (uint32_t)e == awork + 1;
                            live_cut = max(live_cut, (int64_t)(e >> 32));
                        }
                        if (all && t >= live_cut) {
                            mbar_wait(bar_empty + 8 * stage, phase ^ 1, p.stats, p.hdbg);
                            sStop[stage] = 1u;
                            mbar_arrive(bar_full + 8 * stage);              // release: the flag is visible to the waiters
                            if (++stage == S) { stage = 0; phase ^= 1; }
                            break;
                        }
                    }
                    for (int sl = 0; sl < KA; ++sl) {
                        // K slab `sl` of item tile t (the atoms of a packed tile are contiguous)
                        const unsigned char* src = reinterpret_cast<const unsigned char*>(p.Bp) + (size_t)t * p.b_bytes +
                                                   (size_t)sl * STAGE_BYTES;
                        mbar_wait(bar_empty + 8 * stage, phase ^ 1, p.stats, p.hdbg);
                        sStop[stage] = 0u;
                        mbar_arrive_expect_tx(bar_full + 8 * stage, STAGE_BYTES);
                        bulk_g2s(smem_u32(sB + (size_t)stage * STAGE_BYTES), src, STAGE_BYTES, bar_full + 8 * stage);
                        if (++stage == S) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else {
        // ============================ consumers =====================================
        // Warpgroup wg multiplies users [64 wg, 64 wg + 64) of the tile.  In the accumulator layout a quad of lanes holds
        // two users (rows r and r + 8) and all 128 items between them; lane q of the quad owns row r + 8 (q >> 1) and the
        // item half h = q & 1 (32-column chunks 2h, 2h + 1).  Each (user, half) keeps its own candidate list.
        const int wg = warp >> 2;
        const int q = lane & 3, h = q & 1;
        const int row = wg * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * (q >> 1);
        const int etid = tid;                                  // 0..255 = 32 warp + lane
        // byte offset of this row's threshold pair inside the packed A tile
        const uint32_t thr_off = (uint32_t)tile_byte(BM, row, p.rs);
        const bool vec_ok = ((p.lde | p.ldv) % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.E) | reinterpret_cast<uintptr_t>(p.V)) % 16 == 0);
        const uint64_t adesc0 = gmma_desc_sw128(smem_u32(sA) + (uint32_t)wg * 64 * 128);
        const uint64_t bdesc0 = gmma_desc_sw128(smem_u32(sB));
        uint32_t awork = 0, gslab = 0;           // gslab: ring stages consumed so far (the producer fills them in this order)
        unsigned long long n_rescored = 0, n_swept = 0;
        uint32_t my_gen = 0;
        for (int64_t wi = 0; next_work(p, wi, cta, n_ctas, n_groups, wk); ++wi, ++awork) {
            const int64_t ut = wk.g; const int part = wk.part;
            const int64_t t_lo = min(p.item_tiles, p.tile_first + (int64_t)part * p.tiles_per_part);
            int64_t t_hi = min(p.item_tiles, p.tile_first + (int64_t)(part + 1) * p.tiles_per_part);
            if (p.need_sorted) t_hi = min(t_hi, max(t_lo, (int64_t)__ldg(p.need_sorted + wk.g * BM)));
            const int64_t tr = ut * BM + row;                              // tile row
            const bool live = tr < p.m;
            const int64_t u = (live && p.uperm) ? (int64_t)__ldg(p.uperm + tr) : tr;     // user id
            ListState ls;
            ls.list = p.lists + ((int64_t)(part * 2 + h) * p.m + (live ? u : 0)) * p.k;
            ls.cnt = 0; ls.kth = -CUDART_INF_F;
            if (live) for (int j = 0; j < p.k; ++j) { pb200_cand c; c.score = -CUDART_INF_F; c.id = -1; ls.list[j] = c; }
            float t_row = live ? __ldg(p.t0 + u) : CUDART_INF_F;           // best known lower bound of the k-th score
            float t_written = t_row;
            const float* erow = p.E + (live ? u : 0) * p.lde;
            int64_t sb = 0, se = 0;                                        // this user's seen list (sorted item ids)
            if (live && p.seen_indptr) { sb = p.seen_indptr[u]; se = p.seen_indptr[u + 1]; }
            const uint32_t* head = (live && p.headbits) ? p.headbits + u * HEAD_WORDS : nullptr;
            int scount = 0;
            mbar_wait(bar_afull, awork & 1, p.stats, p.hdbg);                              // A tile (and its threshold slots) landed
            // live cut: the item tile from which this row needs nothing under t_row (first_cut_tile; 0 for padding rows),
            // published as the maximum over the warp.  It starts at the row's cut under t0 and falls as t_row rises.
            int cut_row = 0;
            auto publish_cut = [&](int64_t t_next) {
                if (live && cut_row > t_next) {
                    // search only when the cut moves: the bound at the start of the last needed tile fell below t_row
                    const float en = __ldg(p.enorm + u);
                    if (en * __ldg(p.vnorm_sorted + (int64_t)(cut_row - 1) * BN) < t_row)
                        cut_row = first_cut_tile(en, t_row, p.vnorm_sorted, (int)t_next, cut_row - 1);
                }
                const int wcut = __reduce_max_sync(0xffffffffu, cut_row);
                if (lane == 0) sCut[warp] = ((unsigned long long)(uint32_t)wcut << 32) | (unsigned long long)(awork + 1);
            };
            if (p.need_sorted) {
                cut_row = live ? __ldg(p.need_sorted + tr) : 0;
                publish_cut(t_lo);
            }

            auto flush = [&]() {
                {
                    int nsurv = 0;
                    for (int e = 0; e < scount; ++e) nsurv += __popc(sStage[e * 256 + etid].y);
                    uint32_t big = __ballot_sync(0xffffffffu, live && nsurv >= COOP_MIN);
                    if (big) {
                        __syncwarp();                              // the owners' list entries are visible to the warp
                        do {
                            const int src = __ffs(big) - 1;
                            big &= big - 1;
                            const int64_t u_s = __shfl_sync(0xffffffffu, u, src);
                            const int64_t sb_s = __shfl_sync(0xffffffffu, sb, src), se_s = __shfl_sync(0xffffffffu, se, src);
                            const int n_s = __shfl_sync(0xffffffffu, scount, src);
                            const float t_s = __shfl_sync(0xffffffffu, t_row, src);
                            const int h_s = __shfl_sync(0xffffffffu, h, src);
                            int cnt_s = __shfl_sync(0xffffffffu, ls.cnt, src);
                            float kth_s = __shfl_sync(0xffffffffu, ls.kth, src);
                            CoopArgs ca;
                            ca.V = p.V; ca.ldv = p.ldv; ca.perm = p.perm; ca.seen_indices = p.seen_indices;
                            ca.seen_offset = p.seen_offset; ca.n = p.n; ca.r = p.r; ca.k = p.k;
                            n_rescored += (unsigned long long)coop_flush_row(
                                ca, p.E + u_s * p.lde, sStage + (etid - lane + src), n_s, t_lo, sb_s, se_s, p.headbits != nullptr,
                                p.lists + ((int64_t)(part * 2 + h_s) * p.m + u_s) * p.k, t_s, vec_ok, lane, cnt_s, kth_s);
                            if (lane == src) { ls.cnt = cnt_s; ls.kth = kth_s; scount = 0; }
                        } while (big);
                        __syncwarp();
                    }
                }
                for (int e = 0; e < scount; ++e) {
                    uint2 ent = sStage[e * 256 + etid];
                    const int64_t base = (int64_t)(t_lo + (ent.x >> 2)) * BN + (ent.x & 3) * 32;
                    uint32_t mask = ent.y;
                    while (mask) {
                        int c = __clz(mask);                   // column c <-> bit 31-c (first column packed first)
                        mask &= ~(0x80000000u >> c);
                        const int64_t pos = base + c;
                        if (pos >= p.n) continue;
                        const int64_t item = __ldg(p.perm + pos);          // sweep position -> item id
                        // positions inside the head were masked by the bitmap already
                        if (sb < se && (head == nullptr || pos >= HEAD_TILES * BN) &&
                            seen_lookup(p.seen_indices, sb, se, (int)(item + p.seen_offset))) continue;
                        const float* vrow = p.V + item * p.ldv;
                        const float s = exact_score_vec(erow, vrow, p.r, vec_ok);
                        ++n_rescored;
                        if (s < t_row) continue;               // cannot be in the final top-k
                        list_insert(ls, p.k, s, (int)item);
                    }
                }
                scount = 0;
                // share the per-half k-th scores of this row; both are lower bounds of the final k-th score
                // one 8-byte store / load per entry: {tag (valid for this work item only), k-th score} never tear
                volatile unsigned long long* thr64 = reinterpret_cast<volatile unsigned long long*>(const_cast<uint2*>(sThr));
                thr64[h * 128 + row] = ((unsigned long long)__float_as_uint(ls.kth) << 32) | (unsigned long long)(awork + 1);
                const unsigned long long oent = thr64[(1 - h) * 128 + row];
                const uint32_t otag = (uint32_t)oent;
                const float oval = __uint_as_float((uint32_t)(oent >> 32));
                // the other half may be one update behind or ahead; any value carrying this work's tag
                // is the k-th score of k real unseen items of this user, hence a valid lower bound
                const float other = (otag == awork + 1) ? oval : -CUDART_INF_F;
                t_row = fmaxf(t_row, fmaxf(ls.kth, other));
                if (live && t_row > t_written) {
                    // both halves of a row may write: each writes a valid lower bound
                    *reinterpret_cast<volatile uint32_t*>(sA + thr_off) = pack_threshold(t_row);
                    t_written = t_row;
                    fence_proxy_async();                       // make the generic-proxy store visible to the wgmma reads
                }
            };

            const int ntiles = (int)(t_hi - t_lo);
            int j = 0;
            for (; j < ntiles; ++j) {
                const int64_t t = t_lo + j;
                if (p.need_sorted) {
                    // the producer may have ended the sweep here (live cut): that stage only carries the flag
                    const uint32_t st = gslab % S, ph = (gslab / S) & 1u;
                    mbar_wait(bar_full + 8 * st, ph, p.stats, p.hdbg);
                    if (sStop[st]) {
                        ++gslab;
                        __syncwarp();
                        if (lane == 0) mbar_arrive(bar_empty + 8 * st);
                        break;
                    }
                }
                // ---- D = A_wg B_t^T over the K slabs of the tile; a stage goes back to the producer when its MMAs retired
                float d[64];
#pragma unroll
                for (int i = 0; i < 64; ++i) d[i] = 0.f;
                uint32_t prev = 0;
                for (int sl = 0; sl < KA; ++sl) {
                    const uint32_t st = gslab % S, ph = (gslab / S) & 1u;
                    ++gslab;
                    mbar_wait(bar_full + 8 * st, ph, p.stats, p.hdbg);
                    wg_fence_acc(d);
                    wg_fence();
                    // all four K steps of the slab: the packed atoms are zero beyond KP, and a wgmma under a data-dependent
                    // branch makes ptxas serialize every wgmma of the kernel (C7520)
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks)
                        wgmma_m64n128k16(d, adesc0 + (uint64_t)((uint32_t)sl * (BM * 128 / 16) + (uint32_t)ks * 2),
                                         bdesc0 + (uint64_t)(st * (STAGE_BYTES / 16) + (uint32_t)ks * 2), (sl | ks) != 0);
                    wg_commit();
                    wg_fence_acc(d);
                    if (sl > 0) {
                        wg_wait<1>();
                        __syncwarp();
                        if (lane == 0) mbar_arrive(bar_empty + 8 * prev);
                    }
                    prev = st;
                }
                wg_wait<0>();
                wg_fence_acc(d);
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_empty + 8 * prev);

                // ---- sign bits -> per-row candidate masks.  Word (a, c): row r + 8a, chunk c (columns 32c .. 32c + 31),
                // column 32c + x <-> bit 31 - x; this lane contributes columns 8i + 2q + b, the quad ORs its four parts.
                uint32_t w[2][4];
#pragma unroll
                for (int a = 0; a < 2; ++a)
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        uint32_t mk = 0;
#pragma unroll
                        for (int i = 0; i < 4; ++i)
#pragma unroll
                            for (int b = 0; b < 2; ++b)
                                mk |= (__float_as_uint(d[4 * (4 * c + i) + 2 * a + b]) >> 31) << (31 - 8 * i - b);
                        mk >>= 2 * q;
                        mk |= __shfl_xor_sync(0xffffffffu, mk, 1);
                        mk |= __shfl_xor_sync(0xffffffffu, mk, 2);
                        w[a][c] = mk;
                    }
                const bool hi_row = (q >> 1) != 0;
                uint32_t m0 = hi_row ? (h ? w[1][2] : w[1][0]) : (h ? w[0][2] : w[0][0]);
                uint32_t m1 = hi_row ? (h ? w[1][3] : w[1][1]) : (h ? w[0][3] : w[0][1]);
                // seen items in the head of the sweep order are masked here, before they become candidates
                if (head && t < HEAD_TILES) {
                    const uint2 hb = __ldg(reinterpret_cast<const uint2*>(head + (int)t * (BN / 32) + 2 * h));
                    m0 &= ~hb.x; m1 &= ~hb.y;
                }
                const uint32_t code = (uint32_t)j << 2;
                if (m0 && live) { sStage[scount * 256 + etid] = make_uint2(code | (uint32_t)(2 * h), m0); ++scount; }
                if (m1 && live) { sStage[scount * 256 + etid] = make_uint2(code | (uint32_t)(2 * h + 1), m1); ++scount; }
                {
                    const uint32_t gen = *flush_gen;
                    const bool need = __any_sync(0xffffffffu, scount > CAPS - 2 || (scount >= 4 && t_row == -CUDART_INF_F));
                    if (need || gen != my_gen) {
                        if (need && gen == my_gen && lane == 0) atomicAdd(const_cast<uint32_t*>(flush_gen), 1u);
                        flush();
                        my_gen = *flush_gen;
                        if (p.need_sorted) publish_cut(t + 1);
                    }
                }
            }
            n_swept += (unsigned long long)j;
            flush();
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_aempty);      // this warp no longer touches the A tile
        }
        if (p.stats && n_rescored) atomicAdd(p.stats + 1, n_rescored);
        if (p.stats && tid == 0 && n_swept) atomicAdd(p.stats + 5, n_swept);      // (user tile, item tile) products swept
    }
    __syncthreads();
}

}  // namespace

int pb_score_tc(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv, int64_t m, int64_t n,
                int r, const int64_t* seen_indptr, const int32_t* seen_indices, int64_t seen_offset, int k,
                int* parts_out, pb200_cand** lists_out, Scratch& sc) {
    const int rs = (r + 1) & ~1;                       // threshold pair, 4-byte aligned
    const int KP = ((rs + 3) + 15) / 16 * 16;         // + threshold hi/lo + margin slot
    const int KA = (KP + 63) / 64;                      // 128-byte swizzle atoms along K
    const uint32_t a_bytes = BM * KA * 128, b_bytes = BN * KA * 128;
    const size_t fixed = (size_t)a_bytes + CAPS * 256 * sizeof(uint2) + 256 * sizeof(uint2) + (2 * MAX_STAGES + 4) * 8 +
                         (NCONS / 32) * 8 + MAX_STAGES * 4 + 1024;      // + live cut entries and stop flags
    int dev_smem = 0;
    PB_CUDA(ctx, cudaDeviceGetAttribute(&dev_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
    const int64_t user_tiles = ceil_div64(m, BM), item_tiles = ceil_div64(n, BN);
    // the A tile (all KA atoms) stays resident; every ring stage holds one 64-wide K slab of an item tile
    const int stages = (int)std::min<int64_t>(MAX_STAGES, ((int64_t)dev_smem - (int64_t)fixed) / STAGE_BYTES);
    if (stages < 2) {
        ctx->err = "tensor-core scoring kernel: rank too large for the shared-memory pipeline (use the simt kernel)";
        return PB200_ENOTIMPL;
    }
    // the PROBE_ITEMS largest-norm items (whole tiles only) are scored exactly by the probe kernel and form
    // each user's first candidate list; the tensor-core sweep starts behind them
    const int64_t n_probe = std::min<int64_t>(PROBE_ITEMS, (n / BN) * BN);
    const int64_t tile_first = n_probe / BN, sweep_tiles = item_tiles - tile_first;
    int parts = (int)std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>(ceil_div64(2 * (int64_t)ctx->num_sms, user_tiles), 64),
                                                              std::max<int64_t>(sweep_tiles, 1)));
    const int64_t tiles_per_part = std::max<int64_t>(1, ceil_div64(sweep_tiles, parts));
    parts = (int)std::max<int64_t>(1, ceil_div64(sweep_tiles, tiles_per_part));

    __nv_bfloat16 *Ap = nullptr, *Bp = nullptr;
    float *enorm = nullptr, *vnorm = nullptr, *vnorm_sorted = nullptr, *t0 = nullptr;
    int32_t *iota = nullptr, *perm = nullptr, *inv_perm = nullptr;
    uint32_t* headbits = nullptr;
    pb200_cand* lists = nullptr;
    PB_TRY(sc.alloc(&Ap, (size_t)user_tiles * BM * KA * 64));
    PB_TRY(sc.alloc(&Bp, (size_t)item_tiles * BN * KA * 64));
    PB_TRY(sc.alloc(&enorm, (size_t)m));
    PB_TRY(sc.alloc(&vnorm, (size_t)n));
    PB_TRY(sc.alloc(&vnorm_sorted, (size_t)n));
    PB_TRY(sc.alloc(&iota, (size_t)n));
    PB_TRY(sc.alloc(&perm, (size_t)n));
    PB_TRY(sc.alloc(&t0, (size_t)m));
    PB_TRY(sc.alloc(&lists, (size_t)(parts * 2 + 1) * m * k));          // + the probe list

    // 1) item norms; sweep order = decreasing norm (stable radix sort; CUB is used for the two orderings only)
    row_norm_kernel<<<(unsigned)ceil_div64(n * 32, 256), 256, 0, ctx->stream>>>(V, ldv, n, r, vnorm, nullptr);
    iota_i32_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, ctx->stream>>>(iota, n);
    {
        size_t temp_bytes = 0;
        PB_CUDA(ctx, cub::DeviceRadixSort::SortPairsDescending(nullptr, temp_bytes, vnorm, vnorm_sorted, iota, perm, (int64_t)n, 0, 32, ctx->stream));
        uint8_t* temp = nullptr;
        PB_TRY(sc.alloc(&temp, temp_bytes));
        PB_CUDA(ctx, cub::DeviceRadixSort::SortPairsDescending(temp, temp_bytes, vnorm, vnorm_sorted, iota, perm, (int64_t)n, 0, 32, ctx->stream));
    }
    // 2) bitmap of seen items inside the head of the sweep order (they would all pass the filter)
    if (seen_indptr) {
        PB_TRY(sc.alloc(&inv_perm, (size_t)n));
        PB_TRY(sc.alloc(&headbits, (size_t)m * HEAD_WORDS));
        invert_perm_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, ctx->stream>>>(perm, n, inv_perm);
        uint32_t* in_head = nullptr;
        const int64_t n_head = std::min<int64_t>(n, (int64_t)HEAD_TILES * BN);
        PB_TRY(sc.alloc(&in_head, (size_t)ceil_div64(n, 32)));
        PB_CUDA(ctx, cudaMemsetAsync(in_head, 0, (size_t)ceil_div64(n, 32) * sizeof(uint32_t), ctx->stream));
        head_items_kernel<<<(unsigned)ceil_div64(n_head, 256), 256, 0, ctx->stream>>>(perm, n_head, in_head);
        head_bitmap_kernel<<<(unsigned)ceil_div64(m * 32, 256), 256, 0, ctx->stream>>>(seen_indptr, seen_indices, seen_offset,
                                                                                     inv_perm, in_head, m, n, headbits);
    }
    // 3) exact probe pass over the largest-norm items seeds a lower bound of every user's k-th best score (and
    //    yields the user norms and, with early termination, each user's need in item tiles)
    const bool prune = ctx->prune != 0;
    int32_t* need = nullptr;
    if (prune) PB_TRY(sc.alloc(&need, (size_t)m));
    {
        PB_CUDA(ctx, cudaFuncSetAttribute(probe_kernel<PROBE_ITEMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ProbeSmem<PROBE_ITEMS>)));
        probe_kernel<PROBE_ITEMS><<<(unsigned)ceil_div64(m, PTU), 256, sizeof(ProbeSmem<PROBE_ITEMS>), ctx->stream>>>(
            E, lde, V, ldv, perm, m, n_probe, r, k, headbits, t0, lists + (size_t)parts * 2 * m * k,
            enorm, vnorm_sorted, (int)item_tiles, ctx->bound_fn ? nullptr : need);
    }
    // 3a) item-sharded job: a bound found on any shard holds for the merged lists (pb200_set_bound_hook)
    if (ctx->bound_fn) {
        const int st = ctx->bound_fn(ctx->bound_user, t0, m, PB200_F32);
        if (st != 0) {
            ctx->err = "bound hook failed with status " + std::to_string(st);
            return PB200_ECUDA;
        }
        if (prune) user_need_kernel<<<(unsigned)ceil_div64(m, 256), 256, 0, ctx->stream>>>(enorm, t0, vnorm_sorted, m, (int)item_tiles, need);
    }
    // 3b) early termination (pb200_set_prune; exact, see first_cut_tile): user tiles are formed from users of similar
    //     need, so a tile sweeps about as far as its users need rather than as far as its neediest one does.  Users
    //     sorted by need, descending: tile rows -> users (uperm); the tiles come out longest first (next_work).
    int32_t *uperm = nullptr, *need_sorted = nullptr;
    if (prune) {
        int32_t* uiota = nullptr;
        PB_TRY(sc.alloc(&uiota, (size_t)m));
        PB_TRY(sc.alloc(&uperm, (size_t)m));
        PB_TRY(sc.alloc(&need_sorted, (size_t)m));
        iota_i32_kernel<<<(unsigned)ceil_div64(m, 256), 256, 0, ctx->stream>>>(uiota, m);
        int end_bit = 1;                                          // need is in [0, item_tiles]
        while (end_bit < 31 && ((int64_t)1 << end_bit) <= item_tiles) ++end_bit;
        size_t temp_bytes = 0;
        PB_CUDA(ctx, cub::DeviceRadixSort::SortPairsDescending(nullptr, temp_bytes, need, need_sorted, uiota, uperm, m, 0, end_bit, ctx->stream));
        uint8_t* temp = nullptr;
        PB_TRY(sc.alloc(&temp, temp_bytes));
        PB_CUDA(ctx, cub::DeviceRadixSort::SortPairsDescending(temp, temp_bytes, need, need_sorted, uiota, uperm, m, 0, end_bit, ctx->stream));
    }
    // 4) operand packing (user norms feed the per-pair margin)
    {
        int64_t tot_b = item_tiles * BN * (KA * 8), tot_a = user_tiles * BM * (KA * 8);
        pack_items_kernel<<<(unsigned)ceil_div64(tot_b, 256), 256, 0, ctx->stream>>>(V, ldv, n, r, rs, KP, item_tiles, perm, vnorm_sorted, Bp);
        pack_users_kernel<<<(unsigned)ceil_div64(tot_a, 256), 256, 0, ctx->stream>>>(E, lde, m, r, rs, KP, user_tiles, uperm, enorm, t0, Ap);
    }
    if (sweep_tiles <= 0) {
        // every item was in the probe set: only the probe list exists
        cudaEventRecord(ctx->ev0, ctx->stream);
        cudaEventRecord(ctx->ev1, ctx->stream);
        *parts_out = 1;
        *lists_out = lists + (size_t)parts * 2 * m * k;
        PB_CUDA(ctx, cudaGetLastError());
        return PB200_OK;
    }
    // 5) the fused tensor-core kernel
    TcParams p;
    p.Ap = Ap; p.Bp = Bp; p.E = E; p.lde = lde; p.V = V; p.ldv = ldv; p.perm = perm; p.t0 = t0;
    p.m = m; p.n = n; p.r = r; p.KP = KP; p.rs = rs; p.k = k;
    p.user_tiles = user_tiles; p.item_tiles = item_tiles; p.parts = parts; p.tiles_per_part = tiles_per_part;
    p.tile_first = tile_first;
    p.seen_indptr = seen_indptr; p.seen_indices = seen_indices; p.seen_offset = seen_offset;
    p.lists = lists; p.stages = stages; p.a_bytes = a_bytes; p.b_bytes = b_bytes;
    p.uperm = uperm; p.need_sorted = need_sorted; p.enorm = enorm; p.vnorm_sorted = vnorm_sorted; p.headbits = headbits;
    p.stats = reinterpret_cast<unsigned long long*>(ctx->d_stats);
    p.hdbg = nullptr;
    if (ctx->h_dbg) {
        unsigned long long* dptr = nullptr;
        if (cudaHostGetDevicePointer(&dptr, ctx->h_dbg, 0) == cudaSuccess) p.hdbg = dptr;
    }
    const size_t smem_bytes = fixed + (size_t)stages * STAGE_BYTES;
    PB_CUDA(ctx, cudaFuncSetAttribute(score_topk_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
    const int64_t n_groups = user_tiles * parts;
    const unsigned grid = (unsigned)std::min<int64_t>(n_groups, ctx->num_sms);
    cudaEventRecord(ctx->ev0, ctx->stream);
    score_topk_tc_kernel<<<grid, NTHREADS, smem_bytes, ctx->stream>>>(p);
    cudaEventRecord(ctx->ev1, ctx->stream);
    ctx->stats[0] += (seen_indptr ? 13 : 10) + (prune ? 2 : 0) + (prune && ctx->bound_fn ? 1 : 0);
    ctx->stats[2] = (uint64_t)item_tiles; ctx->stats[3] = (uint64_t)user_tiles;
    ctx->stats[6] += (uint64_t)(user_tiles * sweep_tiles);   // what [5] would grow by without the early termination
    PB_CUDA(ctx, cudaGetLastError());
    *parts_out = parts * 2 + 1;
    *lists_out = lists;
    return PB200_OK;
}

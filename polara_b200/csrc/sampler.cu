// On-the-fly sampling of unseen items for the sampled evaluation protocol (RandomSampleEvaluationSVDMixin,
// polara/recommender/models.py:1137-1183), reproducing the reference's draws bit for bit:
//   pb200_sample_unseen   sample_row_wise (polara/lib/sampler.py:96-111): the item ids only;
//   pb200_sampled_topk    mf_random_item_scoring (sampler.py:73-93) + the concatenation with the holdout scores and the
//                         per-row topsort (models.py:1178-1183), fused: no [m x (h + n_samples)] block reaches HBM;
//   pb200_sampled_topk_ranks  the same at several truncated ranks of one factor pair (find_optimal_svd_rank,
//                         evaluation/pipelines.py:81-116): one draw per user, one score chain per item, one list per rank.
//
// The reference, per user: numba's random.seed(seed) (MT19937 init_genrand), prime_sampler_state (excluded items moved
// to the tail of range(n) in LIST order through two dicts, `state` position -> item and `track` item -> position), then
// n_samples times i = randrange(remaining) (CPython rule: b = bit_length(remaining), w >> (32 - b) of a raw word,
// redrawn while >= remaining), item = state.get(i, i), remaining -= 1, state[i] = state.get(remaining, remaining),
// state.pop(remaining).  Here one WARP runs one user's chain: the chain is sequential and cannot be split, so lane 0
// does the dict operations and the acceptance test, the warp shares the MT19937 twist (32 words per step; the twist's
// dependencies are 1 and 227 words apart) and, on the fused path, scores the drawn items 32 at a time.
//
// The dicts are one open-addressing table (linear probing, backward-shift deletion: a faithful map, get / set / pop have
// exactly the dict's semantics; iteration order is never used).  `track` keys carry bit 31.  Entries never exceed
// 2 L + n_samples (L = exclusion length): priming adds at most one `state` and one `track` key per excluded item, every
// draw adds at most one `state` key, nothing is dropped early.  A user whose table (map_slots_for) fits the per-warp
// shared-memory budget runs from shared memory, the others from a per-warp table in global memory (same code).
#include "topk_common.cuh"

#include <algorithm>

namespace {

constexpr int MT_N = 624, MT_M = 397;
constexpr int WARPS = 4;                                  // warps (= users in flight) per block
constexpr unsigned long long EMPTY = ~0ull;
constexpr uint32_t TRACK = 0x80000000u;                  // tag of `track` keys (ids are < 2^31)
constexpr int MAX_SMEM_SLOTS = 6144;                      // 4 warps x (2.5 KB MT + 48 KB map) fits one block per SM
constexpr size_t GLOBAL_MAP_BUDGET = size_t(256) << 20;  // bytes of global tables in flight
constexpr size_t GLOBAL_LIST_BUDGET = size_t(256) << 20; // bytes of running lists of the global-path warps
constexpr int MAX_RANKS = 64;                             // ranks per fused call (kept in the kernel parameters)

// table size for a user: the entry bound 2L + s at a load factor <= 2/3, plus a floor
__host__ __device__ __forceinline__ int64_t map_slots_for(int64_t L, int64_t s) {
    const int64_t need = 2 * L + s;
    return need + need / 2 + 32;
}

__device__ __forceinline__ uint32_t home(uint32_t key, uint32_t cap) {
    return (uint32_t)(((uint64_t)(key * 0x9E3779B1u) * cap) >> 32);
}

struct Map {
    unsigned long long* slot;
    uint32_t cap;

    __device__ __forceinline__ uint32_t get(uint32_t key, uint32_t dflt) const {
        uint32_t i = home(key, cap);
        while (true) {
            const unsigned long long e = slot[i];
            if (e == EMPTY) return dflt;
            if ((uint32_t)(e >> 32) == key) return (uint32_t)e;
            if (++i == cap) i = 0;
        }
    }
    __device__ __forceinline__ void set(uint32_t key, uint32_t val) const {
        uint32_t i = home(key, cap);
        while (true) {
            const unsigned long long e = slot[i];
            if (e == EMPTY || (uint32_t)(e >> 32) == key) break;
            if (++i == cap) i = 0;
        }
        slot[i] = ((unsigned long long)key << 32) | val;
    }
    __device__ __forceinline__ void pop(uint32_t key) const {
        uint32_t i = home(key, cap);
        while (true) {
            const unsigned long long e = slot[i];
            if (e == EMPTY) return;
            if ((uint32_t)(e >> 32) == key) break;
            if (++i == cap) i = 0;
        }
        // backward shift: pull later entries of the probe run into the hole unless their home lies in (hole, j]
        uint32_t j = i;
        while (true) {
            if (++j == cap) j = 0;
            const unsigned long long e = slot[j];
            if (e == EMPTY) break;
            const uint32_t h = home((uint32_t)(e >> 32), cap);
            const bool stays = (i <= j) ? (h > i && h <= j) : (h > i || h <= j);
            if (stays) continue;
            slot[i] = e;
            i = j;
        }
        slot[i] = EMPTY;
    }
};

// MT19937 twist, warp-parallel in steps of 32 words: word i reads words i+1 (old, or new word 0 for i = 623) and
// i+397 mod 624 (old for i < 227, new for i >= 227 -- written at least 227 words earlier, so in an earlier step)
__device__ __forceinline__ void mt_twist(uint32_t* mt, int lane) {
    for (int base = 0; base < MT_N; base += 32) {
        const int i = base + lane;
        uint32_t nv = 0;
        if (i < MT_N) {
            const uint32_t y = (mt[i] & 0x80000000u) | (mt[i + 1 < MT_N ? i + 1 : 0] & 0x7fffffffu);
            nv = mt[i + MT_M < MT_N ? i + MT_M : i + MT_M - MT_N] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        }
        __syncwarp();
        if (i < MT_N) mt[i] = nv;
        __syncwarp();
    }
}

// next tempered word (warp-uniform: every lane reads the same word)
__device__ __forceinline__ uint32_t mt_next(uint32_t* mt, int& idx, int lane) {
    if (idx >= MT_N) { mt_twist(mt, lane); idx = 0; }
    uint32_t y = mt[idx++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
}

// numba's random.randrange(n), CPython flavour (numba/cpython/randomimpl.py): top bit_length(n) bits, redraw if >= n
__device__ __forceinline__ uint32_t randrange(uint32_t* mt, int& idx, int lane, uint32_t n) {
    const int shift = __clz(n);                           // 32 - bit_length(n); n >= 1
    while (true) {
        const uint32_t r = mt_next(mt, idx, lane) >> shift;
        if (r < n) return r;
    }
}

struct Params {
    int64_t m, n;
    const int64_t* excl_indptr;
    const int32_t* excl_indices;
    const uint32_t* seeds;
    int s;                                                 // samples per user
    // pb200_sample_unseen
    int64_t* out_items;
    int64_t ld_out;
    // pb200_sampled_topk
    const float* E;
    int64_t lde;
    const float* V;
    int64_t ldv;
    int nr;                                                // truncated ranks, strictly ascending
    int ranks[MAX_RANKS];
    const int64_t* holdout;                                // [m x h]
    int h, k;
    int64_t* out_pos;                                      // [nr x m x k], rank-major
    float* out_scores;
    pb200_cand* lists;                                     // [warps in the grid x nr x k] running top-k lists
    // map placement
    int smem_slots;                                        // shared-memory path: slots per warp
    const int64_t* heavy;                                  // global path: users, count, table slots per warp
    int64_t n_heavy;
    unsigned long long* gmaps;
    int64_t gslots;
};

// offer one batch of up to 32 (score, position) pairs, lane t holding position base + t (ascending), to the running
// top-k list: the filter and order of pb200_topk_dense ((score desc, position asc); NaN never enters)
__device__ __forceinline__ void offer(pb200_cand* list, int k, int& cnt, float& thr, bool have, float x, int pos, int lane) {
    const bool pass = have && ((cnt < k) ? (x == x) : (x > thr));
    unsigned mask = __ballot_sync(0xffffffffu, pass);
    while (mask) {
        const int t = __ffs(mask) - 1;
        mask &= mask - 1;
        cnt = warp_list_insert(list, k, cnt, __shfl_sync(0xffffffffu, x, t), __shfl_sync(0xffffffffu, pos, t), lane);
        if (cnt == k) thr = list[k - 1].score;
    }
}

// exact_score's chain continued over columns [t0, t1)
__device__ __forceinline__ float score_chain(const float* __restrict__ e, const float* __restrict__ v, int t0, int t1,
                                             float s) {
    for (int t = t0; t < t1; ++t) s = fmaf(e[t], v[t], s);
    return s;
}

// One batch of up to 32 items, lane t holding item `item` (valid if `have`) at row position `pos`, offered to the list
// of every rank: the lane's score chain fmaf(e[t], v[t], s), t ascending from 0, is continued from ranks[j-1] to
// ranks[j] before list j sees it, so list j gets exactly exact_score(e, v, ranks[j]) and each V row is read once.  Ids
// out of [0, n) score NaN at every rank and never enter.  List 0's fill and threshold are plain registers (cnt0 / thr0:
// the single-rank call keeps the code it had; read back through a shuffle, they are no longer known to be warp-uniform
// and the list insertions run ~5 % slower); list j >= 1's live in lane j % 32 of cnt_lo/thr_lo (j < 32) or
// cnt_hi/thr_hi, out of local memory.
__device__ __forceinline__ void offer_ranks(const Params& p, const float* e, pb200_cand* lists, int& cnt0, float& thr0,
                                            int& cnt_lo, int& cnt_hi, float& thr_lo, float& thr_hi, bool have, int64_t item,
                                            int pos, int lane) {
    const bool valid = have && item >= 0 && item < p.n;
    const float* v = p.V + (valid ? item : 0) * p.ldv;
    int t = p.ranks[0];
    float s = valid ? score_chain(e, v, 0, t, 0.f) : 0.f;
    offer(lists, p.k, cnt0, thr0, have, valid ? s : CUDART_NAN_F, pos, lane);
    for (int j = 1; j < p.nr; ++j) {
        const int rj = p.ranks[j];
        if (valid) s = score_chain(e, v, t, rj, s);
        t = rj;
        const bool hi = j >= 32;
        int cnt = __shfl_sync(0xffffffffu, hi ? cnt_hi : cnt_lo, j & 31);
        float thr = __shfl_sync(0xffffffffu, hi ? thr_hi : thr_lo, j & 31);
        offer(lists + (int64_t)j * p.k, p.k, cnt, thr, have, valid ? s : CUDART_NAN_F, pos, lane);
        if (lane == (j & 31)) {
            if (hi) { cnt_hi = cnt; thr_hi = thr; } else { cnt_lo = cnt; thr_lo = thr; }
        }
    }
}

template <bool FUSED>
__device__ void run_user(const Params& p, int64_t u, uint32_t* mt, Map map, pb200_cand* lists, int lane) {
    const int64_t b = p.excl_indptr[u], L = p.excl_indptr[u + 1] - b;
    // random.seed(seeds[u]): init_genrand
    if (lane == 0) {
        uint32_t x = p.seeds[u];
        mt[0] = x;
        for (int i = 1; i < MT_N; ++i) {
            x = 1812433253u * (x ^ (x >> 30)) + (uint32_t)i;
            mt[i] = x;
        }
    }
    for (uint32_t i = lane; i < map.cap; i += 32) map.slot[i] = EMPTY;
    __syncwarp();
    // prime_sampler_state: excluded items, in list order, to the tail
    const uint32_t last = (uint32_t)(p.n - 1);
    for (int64_t c0 = 0; c0 < L; c0 += 32) {
        const uint32_t mine = (c0 + lane < L) ? (uint32_t)p.excl_indices[b + c0 + lane] : 0u;
        const int cn = L - c0 < 32 ? (int)(L - c0) : 32;
        for (int t = 0; t < cn; ++t) {
            const uint32_t item = __shfl_sync(0xffffffffu, mine, t);
            if (lane == 0) {
                const uint32_t pos = last - (uint32_t)(c0 + t);
                const uint32_t x = map.get(TRACK | item, item);
                const uint32_t tv = map.get(pos, pos);
                map.set(x, tv);
                map.set(TRACK | tv, x);
                map.pop(pos);
                map.pop(TRACK | item);
            }
        }
    }
    __syncwarp();
    int cnt0 = 0, cnt_lo = 0, cnt_hi = 0;
    float thr0 = -CUDART_INF_F, thr_lo = -CUDART_INF_F, thr_hi = -CUDART_INF_F;
    const float* e = nullptr;
    if (FUSED) {
        e = p.E + u * p.lde;
        // holdout items first: positions 0 .. h-1 (pb200_gather_dot's scores: NaN for ids out of range)
        for (int c0 = 0; c0 < p.h; c0 += 32) {
            const int j = c0 + lane;
            const int64_t it = j < p.h ? p.holdout[u * p.h + j] : -1;
            offer_ranks(p, e, lists, cnt0, thr0, cnt_lo, cnt_hi, thr_lo, thr_hi, j < p.h, it, j, lane);
        }
    }
    // sample_fill
    uint32_t remaining = (uint32_t)(p.n - L);
    int idx = MT_N;
    uint32_t held = 0;                                     // fused: lane t holds the draw of batch slot t
    for (int j = 0; j < p.s; ++j) {
        const uint32_t i = randrange(mt, idx, lane, remaining);
        uint32_t item = 0;
        --remaining;
        if (lane == 0) {
            item = map.get(i, i);
            map.set(i, map.get(remaining, remaining));
            map.pop(remaining);
            if (!FUSED) p.out_items[u * p.ld_out + j] = (int64_t)item;
        }
        if (FUSED) {
            item = __shfl_sync(0xffffffffu, item, 0);
            if (lane == (j & 31)) held = item;
            if ((j & 31) == 31 || j == p.s - 1) {
                const int c0 = j & ~31;
                offer_ranks(p, e, lists, cnt0, thr0, cnt_lo, cnt_hi, thr_lo, thr_hi, c0 + lane <= j, (int64_t)held,
                            p.h + c0 + lane, lane);
            }
        }
    }
    if (FUSED) {
        __syncwarp();
        for (int j = 0; j < p.nr; ++j) {
            const int cnt = j == 0 ? cnt0 : __shfl_sync(0xffffffffu, j >= 32 ? cnt_hi : cnt_lo, j & 31);
            const pb200_cand* list = lists + (int64_t)j * p.k;
            const int64_t o = ((int64_t)j * p.m + u) * p.k;
            for (int i = lane; i < p.k; i += 32) {
                const bool ok = i < cnt;
                p.out_pos[o + i] = ok ? (int64_t)list[i].id : -1;
                if (p.out_scores) p.out_scores[o + i] = ok ? list[i].score : -CUDART_INF_F;
            }
        }
        __syncwarp();
    }
}

// users whose table fits in the shared-memory budget; the others are left to sampler_gmem_kernel
template <bool FUSED>
__global__ void __launch_bounds__(WARPS * 32) sampler_smem_kernel(Params p) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const size_t per_warp = MT_N * sizeof(uint32_t) + (size_t)p.smem_slots * sizeof(unsigned long long);
    uint32_t* mt = reinterpret_cast<uint32_t*>(smem + w * per_warp);
    unsigned long long* slots = reinterpret_cast<unsigned long long*>(mt + MT_N);
    const int64_t gw = (int64_t)blockIdx.x * WARPS + w, nw = (int64_t)gridDim.x * WARPS;
    pb200_cand* lists = FUSED ? p.lists + gw * p.nr * p.k : nullptr;
    for (int64_t u = gw; u < p.m; u += nw) {
        const int64_t L = p.excl_indptr[u + 1] - p.excl_indptr[u];
        const int64_t cap = map_slots_for(L, p.s);
        if (cap > p.smem_slots) continue;
        run_user<FUSED>(p, u, mt, Map{slots, (uint32_t)cap}, lists, lane);
    }
}

// users whose table does not fit: one table of p.gslots slots per warp in global memory.  The minimum block counts hold
// each variant at the register count it needs without spilling (left alone, ptxas caps the fused one at 56 and spills;
// it needs 80)
template <bool FUSED>
__global__ void __launch_bounds__(WARPS * 32, FUSED ? 6 : 10) sampler_gmem_kernel(Params p) {
    __shared__ uint32_t mts[WARPS][MT_N];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t gw = (int64_t)blockIdx.x * WARPS + w, nw = (int64_t)gridDim.x * WARPS;
    pb200_cand* lists = FUSED ? p.lists + gw * p.nr * p.k : nullptr;
    unsigned long long* slots = p.gmaps + gw * p.gslots;
    for (int64_t t = gw; t < p.n_heavy; t += nw) {
        const int64_t u = p.heavy[t];
        const int64_t L = p.excl_indptr[u + 1] - p.excl_indptr[u];
        run_user<FUSED>(p, u, mts[w], Map{slots, (uint32_t)map_slots_for(L, p.s)}, lists, lane);
    }
}

// flags: [0] smallest user with fewer than s items left, [1] smallest user with an id out of range (both ~0 if none),
// [2] users whose table exceeds smem_slots (listed in `heavy`), [3] the largest such table
__global__ void sampler_check_kernel(int64_t m, int64_t n, int s, const int64_t* __restrict__ indptr,
                                     const int32_t* __restrict__ indices, int smem_slots,
                                     unsigned long long* __restrict__ flags, int64_t* __restrict__ heavy) {
    const int lane = threadIdx.x & 31;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t u = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < m; u += nw) {
        const int64_t b = indptr[u], L = indptr[u + 1] - b;
        if (L < 0 || n - L < s) {
            if (lane == 0) atomicMin(flags, (unsigned long long)u);
            continue;
        }
        bool bad = false;
        for (int64_t q = lane; q < L; q += 32) {
            const int32_t x = __ldg(indices + b + q);
            bad |= x < 0 || x >= n;
        }
        if (__any_sync(0xffffffffu, bad)) {
            if (lane == 0) atomicMin(flags + 1, (unsigned long long)u);
            continue;
        }
        const int64_t cap = map_slots_for(L, s);
        if (lane == 0 && cap > smem_slots) {
            heavy[atomicAdd(flags + 2, 1ull)] = u;
            atomicMax(flags + 3, (unsigned long long)cap);
        }
    }
}

int sampler_run(pb200_ctx* ctx, Params p, bool fused) {
    Scratch sc(ctx);
    ctx->sampler_stats[0] = ctx->sampler_stats[1] = ctx->sampler_stats[2] = ctx->sampler_stats[3] = 0;
    p.smem_slots = ctx->sampler_map_slots;
    unsigned long long* flags = nullptr;
    int64_t* heavy = nullptr;
    PB_TRY(sc.alloc(&flags, 4));
    PB_TRY(sc.alloc(&heavy, (size_t)p.m));
    PB_CUDA(ctx, cudaMemsetAsync(flags, 0xff, 2 * sizeof(unsigned long long), ctx->stream));
    PB_CUDA(ctx, cudaMemsetAsync(flags + 2, 0, 2 * sizeof(unsigned long long), ctx->stream));
    const unsigned cblocks = (unsigned)std::min<int64_t>(ceil_div64(p.m * 32, 256), 32 * (int64_t)ctx->num_sms);
    sampler_check_kernel<<<cblocks, 256, 0, ctx->stream>>>(p.m, p.n, p.s, p.excl_indptr, p.excl_indices, p.smem_slots,
                                                          flags, heavy);
    PB_CUDA(ctx, cudaGetLastError());
    unsigned long long hf[4];
    PB_CUDA(ctx, cudaMemcpyAsync(hf, flags, sizeof hf, cudaMemcpyDeviceToHost, ctx->stream));
    PB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->stats[0] += 1;
    ctx->sampler_stats[3] = 1;
    if (hf[0] != ~0ull) {
        ctx->err = "invalid argument: sample_unseen: user " + std::to_string(hf[0]) + " has fewer than " +
                   std::to_string(p.s) + " items left to sample (empty range for randrange())";
        return PB200_EINVAL;
    }
    if (hf[1] != ~0ull) {
        ctx->err = "invalid argument: sample_unseen: exclusion list of user " + std::to_string(hf[1]) +
                   " holds an item id outside [0, n_items)";
        return PB200_EINVAL;
    }
    const int64_t n_heavy = (int64_t)hf[2];
    ctx->sampler_stats[0] = (uint64_t)(p.m - n_heavy);
    ctx->sampler_stats[1] = (uint64_t)n_heavy;
    if (p.s == 0 && !fused) return PB200_OK;
    int dev_max_blocks = 0;
    if (n_heavy < p.m) {
        const size_t smem = WARPS * (MT_N * sizeof(uint32_t) + (size_t)p.smem_slots * sizeof(unsigned long long));
        auto kern = fused ? sampler_smem_kernel<true> : sampler_smem_kernel<false>;
        PB_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        PB_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&dev_max_blocks, kern, WARPS * 32, smem));
        const int64_t blocks = std::max<int64_t>(1, std::min<int64_t>(ceil_div64(p.m, WARPS),
                                                                      (int64_t)std::max(dev_max_blocks, 1) * ctx->num_sms));
        if (fused) PB_TRY(sc.alloc(&p.lists, (size_t)blocks * WARPS * p.nr * p.k));
        kern<<<(unsigned)blocks, WARPS * 32, smem, ctx->stream>>>(p);
        PB_CUDA(ctx, cudaGetLastError());
        ctx->stats[0] += 1;
        ctx->sampler_stats[3] += 1;
    }
    if (n_heavy > 0) {
        const int64_t gslots = (int64_t)hf[3];
        PB_REQUIRE(ctx, gslots < (int64_t)UINT32_MAX, "sample_unseen: exclusion list too long");
        const int64_t by_mem = std::max<int64_t>(1, (int64_t)(GLOBAL_MAP_BUDGET / ((size_t)gslots * 8)));
        const int64_t by_lists = fused ? std::max<int64_t>(1, (int64_t)(GLOBAL_LIST_BUDGET / ((size_t)p.nr * p.k *
                                                                                                sizeof(pb200_cand))))
                                       : n_heavy;
        const int64_t warps = std::min<int64_t>({n_heavy, by_mem, by_lists, (int64_t)ctx->num_sms * 16 * WARPS});
        const int64_t blocks = ceil_div64(warps, WARPS);
        p.heavy = heavy;
        p.n_heavy = n_heavy;
        p.gslots = gslots;
        PB_TRY(sc.alloc(&p.gmaps, (size_t)blocks * WARPS * gslots));
        if (fused) PB_TRY(sc.alloc(&p.lists, (size_t)blocks * WARPS * p.nr * p.k));
        auto kern = fused ? sampler_gmem_kernel<true> : sampler_gmem_kernel<false>;
        kern<<<(unsigned)blocks, WARPS * 32, 0, ctx->stream>>>(p);
        PB_CUDA(ctx, cudaGetLastError());
        ctx->stats[0] += 1;
        ctx->sampler_stats[2] = (uint64_t)gslots;
        ctx->sampler_stats[3] += 1;
    }
    return PB200_OK;
}

}  // namespace

extern "C" int pb200_set_sampler_map_slots(pb200_ctx* ctx, int slots) {
    if (!ctx) return PB200_EINVAL;
    PB_REQUIRE(ctx, slots >= 0 && slots <= MAX_SMEM_SLOTS, "set_sampler_map_slots: slots must be in 0..6144");
    ctx->sampler_map_slots = slots;
    return PB200_OK;
}

extern "C" int pb200_sampler_stats(pb200_ctx* ctx, uint64_t* out4_host) {
    if (!ctx || !out4_host) return PB200_EINVAL;
    for (int i = 0; i < 4; ++i) out4_host[i] = ctx->sampler_stats[i];
    return PB200_OK;
}

extern "C" int pb200_sample_unseen(pb200_ctx* ctx, int64_t m, int64_t n_items, const int64_t* excl_indptr,
                                   const int32_t* excl_indices, const uint32_t* seeds_u32, int n_samples,
                                   int64_t* out_items, int64_t ld_out) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, m >= 0 && n_items > 0 && n_items < (int64_t)2147483647, "sample_unseen: bad shape");
    PB_REQUIRE(ctx, n_samples >= 0 && ld_out >= n_samples, "sample_unseen: need 0 <= n_samples <= ld_out");
    if (m == 0) return PB200_OK;
    PB_REQUIRE(ctx, excl_indptr && excl_indices && seeds_u32 && (out_items || n_samples == 0), "sample_unseen: null argument");
    Params p{};
    p.m = m; p.n = n_items; p.excl_indptr = excl_indptr; p.excl_indices = excl_indices; p.seeds = seeds_u32;
    p.s = n_samples; p.out_items = out_items; p.ld_out = ld_out;
    return sampler_run(ctx, p, false);
}

// pb200_sampled_topk / pb200_sampled_topk_ranks: one routine; the single-rank entry is the rank list {r}
static int sampled_topk_run(pb200_ctx* ctx, const char* where, const float* E, int64_t lde, const float* V, int64_t ldv,
                     int64_t m, int64_t n, const int* ranks, int n_ranks, const int64_t* holdout_items, int h,
                     const int64_t* excl_indptr, const int32_t* excl_indices, const uint32_t* seeds_u32, int n_samples,
                     int k, int64_t* out_pos, float* out_scores) {
    const std::string w(where);
    PB_REQUIRE(ctx, m >= 0 && n > 0 && n < (int64_t)2147483647 && lde > 0 && ldv > 0, (w + ": bad shape").c_str());
    PB_REQUIRE(ctx, h >= 0 && n_samples >= 0, (w + ": negative holdout or sample size").c_str());
    PB_REQUIRE(ctx, k >= 1 && (int64_t)k <= (int64_t)h + n_samples, (w + ": k must be in 1..h + n_samples").c_str());
    Params p{};
    p.nr = n_ranks;
    for (int j = 0; j < n_ranks; ++j) p.ranks[j] = ranks[j];
    if (m == 0) return PB200_OK;
    PB_REQUIRE(ctx, E && V && (holdout_items || h == 0) && excl_indptr && excl_indices && seeds_u32 && out_pos,
               (w + ": null argument").c_str());
    p.m = m; p.n = n; p.excl_indptr = excl_indptr; p.excl_indices = excl_indices; p.seeds = seeds_u32; p.s = n_samples;
    p.E = E; p.lde = lde; p.V = V; p.ldv = ldv; p.holdout = holdout_items; p.h = h; p.k = k;
    p.out_pos = out_pos; p.out_scores = out_scores;
    return sampler_run(ctx, p, true);
}

extern "C" int pb200_sampled_topk(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv, int64_t m,
                                  int64_t n, int r, const int64_t* holdout_items, int h, const int64_t* excl_indptr,
                                  const int32_t* excl_indices, const uint32_t* seeds_u32, int n_samples, int k,
                                  int64_t* out_pos, float* out_scores) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, r > 0 && lde >= r && ldv >= r, "sampled_topk: bad shape");
    return sampled_topk_run(ctx, "sampled_topk", E, lde, V, ldv, m, n, &r, 1, holdout_items, h, excl_indptr,
                            excl_indices, seeds_u32, n_samples, k, out_pos, out_scores);
}

extern "C" int pb200_sampled_topk_ranks(pb200_ctx* ctx, const float* E, int64_t lde, const float* V, int64_t ldv,
                                        int64_t m, int64_t n, const int* ranks_host, int n_ranks,
                                        const int64_t* holdout_items, int h, const int64_t* excl_indptr,
                                        const int32_t* excl_indices, const uint32_t* seeds_u32, int n_samples, int k,
                                        int64_t* out_pos, float* out_scores) {
    PB_ENTER(ctx);
    PB_REQUIRE(ctx, ranks_host && n_ranks >= 1 && n_ranks <= MAX_RANKS,
               "sampled_topk_ranks: the rank list must hold 1..64 ranks");
    for (int j = 0; j < n_ranks; ++j) {
        PB_REQUIRE(ctx, ranks_host[j] >= 1, "sampled_topk_ranks: ranks must be >= 1");
        PB_REQUIRE(ctx, j == 0 || ranks_host[j] > ranks_host[j - 1], "sampled_topk_ranks: ranks must be strictly ascending");
    }
    PB_REQUIRE(ctx, (int64_t)ranks_host[n_ranks - 1] <= lde && (int64_t)ranks_host[n_ranks - 1] <= ldv,
               "sampled_topk_ranks: the largest rank exceeds lde or ldv");
    return sampled_topk_run(ctx, "sampled_topk_ranks", E, lde, V, ldv, m, n, ranks_host, n_ranks, holdout_items, h,
                            excl_indptr, excl_indices, seeds_u32, n_samples, k, out_pos, out_scores);
}

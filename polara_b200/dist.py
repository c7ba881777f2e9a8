"""Item-factor sharding across the GPUs of one box (one process per GPU).

Every rank owns a contiguous slice of the item factors, scores ALL users against its
slice with the fused kernel and emits one sorted candidate list per user; the only
data-path collective is one all-to-all by user range (each rank receives the lists of
"its" users from every peer) followed by a local k-way merge (SURVEY.md §8e).
``torch.distributed`` is plumbing only.
"""
from __future__ import annotations

import torch


class ItemShard:
    """Contiguous item range of this rank plus the user range it owns after the exchange."""

    def __init__(self, rank, world, n_items):
        self.rank, self.world, self.n_items = int(rank), int(world), int(n_items)
        # balanced ranges (sizes differ by at most one): with n_items >= world no rank is left without items, which the
        # scoring kernels refuse (a ceil-sized split gives n = 13, world = 8 the empty range [13, 13) on rank 7)
        if self.n_items < self.world:
            raise ValueError("ItemShard: %d items cannot be split over %d ranks (every rank needs at least one item)"
                             % (self.n_items, self.world))
        self.item_lo = self.rank * self.n_items // self.world
        self.item_hi = (self.rank + 1) * self.n_items // self.world

    def user_chunk(self, n_users):
        """users are split into `world` equal chunks (the last ones may be short/padded)."""
        return (n_users + self.world - 1) // self.world

    def user_range(self, n_users):
        c = self.user_chunk(n_users)
        return min(n_users, self.rank * c), min(n_users, (self.rank + 1) * c)


def max_over_ranks(t):
    """bound hook of item-sharded scoring: a lower bound of a user's k-th best score found on any shard holds everywhere"""
    import torch.distributed as dist
    dist.all_reduce(t, op=dist.ReduceOp.MAX)


def exchange_candidates(cands, world, group=None):
    """``cands`` [m_pad, k, 2] int32 view of {score,id} lists for ALL users (m_pad divisible by
    world) -> [world, m_pad/world, k, 2]: for this rank's user chunk, the lists of every peer."""
    import torch.distributed as dist
    m_pad = cands.shape[0]
    assert m_pad % world == 0
    out = torch.empty_like(cands)
    try:
        dist.all_to_all_single(out, cands, group=group)
    except RuntimeError:
        # backends without all-to-all (CPU tests): same result via all-gather
        gathered = [torch.empty_like(cands) for _ in range(world)]
        dist.all_gather(gathered, cands, group=group)
        rank = dist.get_rank(group)
        chunk = m_pad // world
        out = torch.stack([g[rank * chunk:(rank + 1) * chunk] for g in gathered]).reshape(cands.shape)
    return out.view(world, m_pad // world, *cands.shape[1:])


def row_block(eng, p_dev, shard: ItemShard):
    """this rank's block of user rows of a device CSR as a CSR of its own (row pointers re-based, index/value arrays are
    views): the operand of the row-sharded user-embedding SpMM."""
    from .engine import DeviceCSR
    n_users = p_dev.shape[0]
    lo, hi = shard.user_range(n_users)
    a, b = int(p_dev.indptr[lo]), int(p_dev.indptr[hi])
    ip = p_dev.indptr[lo:hi + 1].clone()
    eng.shift_i64(ip, -a)
    return DeviceCSR(ip, p_dev.indices[a:b], p_dev.values[a:b], (hi - lo, p_dev.shape[1]))


def gather_embeddings(eng, p_block, v_dev, shard: ItemShard, n_users, group=None):
    """E = P V computed ONCE per job: every rank multiplies its block of user rows (SpMM against the whole V, which every
    rank holds) and the blocks are all-gathered over NVLink (SURVEY.md 8e) -- instead of every rank redoing the whole
    product.  Returns E [world * chunk x ld] (rows beyond n_users are padding)."""
    import torch.distributed as dist
    chunk = shard.user_chunk(n_users)
    ld = v_dev.shape[1]
    e_blk = eng.zeros((chunk, ld)) if p_block.shape[0] < chunk else eng.empty((chunk, ld))
    eng.spmm(p_block, v_dev, ell=ld, out=e_blk[: p_block.shape[0]])
    e_all = eng.empty((chunk * shard.world, ld))
    dist.all_gather_into_tensor(e_all, e_blk, group=group)
    return e_all


def sharded_topk(eng, e, v_dev, rank_r, topk, seen, shard: ItemShard, n_users):
    """Fused scoring on this rank's item slice + exchange + merge.  Returns int64 ids
    [user_chunk x topk] of the users this rank owns (global item ids)."""
    v_slice = v_dev[shard.item_lo:shard.item_hi]
    chunk = shard.user_chunk(n_users)
    m_pad = chunk * shard.world
    cands = eng.score_topk_cands(e, v_slice, rank_r, topk, seen=seen, item_offset=shard.item_lo, m=n_users,
                                 m_alloc=m_pad, bound_max=max_over_ranks if shard.world > 1 else None)
    recv = exchange_candidates(cands, shard.world)
    return merge_owned(eng, recv, e, v_dev, rank_r, topk, seen, shard, n_users)


def merge_owned(eng, recv, e, v_dev, rank_r, topk, seen, shard: ItemShard, n_users):
    """k-way merge of the received per-shard lists of the users this rank owns; with seen lists also the reference's
    fill-up (fewer than k unseen items over ALL shards -> seen items follow in score order, models.py:517-519), which
    needs these users' embeddings, the whole V and their seen lists -- all present on the owning rank."""
    chunk = shard.user_chunk(n_users)
    if seen is None:
        return eng.merge_cands(recv, shard.world, chunk, topk)
    lo, hi = shard.user_range(n_users)
    if hi <= lo:
        return eng.empty((chunk, topk), torch.int64)
    return eng.merge_cands_fill(recv, shard.world, chunk, hi - lo, topk, e[lo:hi], v_dev, rank_r, (seen[0][lo:hi + 1], seen[1]))


def gather_lists(recs, shard: ItemShard, n_users, device):
    """the per-rank slices of an item-sharded ``get_recommendations()`` (each rank returns the users it owns) assembled
    into the full ``[n_users x topk]`` array on every rank -- what ``model.recommendations`` / ``evaluate()`` need."""
    import numpy as np
    import torch.distributed as dist
    if n_users is None:                      # every user is owned by exactly one rank
        total = torch.tensor([recs.shape[0]], dtype=torch.int64, device=device)
        dist.all_reduce(total)
        n_users = int(total.item())
    chunk = shard.user_chunk(n_users)
    k = recs.shape[1]
    mine = torch.full((chunk, k), -1, dtype=torch.int64, device=device)
    mine[: recs.shape[0]].copy_(torch.from_numpy(np.ascontiguousarray(recs)))
    full = torch.empty((chunk * shard.world, k), dtype=torch.int64, device=device)
    dist.all_gather_into_tensor(full, mine)
    return full[:n_users].cpu().numpy()


def make_step(eng, p_dev, v_dev, rank_r, topk, shard=None, filter_seen=True, phases=None):
    """One device-resident pass of the hot path: SpMM + fused scoring (+ exchange/merge).  With ``phases`` (a list) the
    step appends ``(name, cuda event)`` marks after every phase -- used for the per-phase table, not in timed loops."""
    seen = (p_dev.indptr, p_dev.indices) if filter_seen else None
    n_users = p_dev.shape[0]
    # the SpMM operand: this rank's rows (sharded) or the whole matrix, stored panel-major when V is too large to stay in
    # L2 while it is gathered from (1e6 items x 128 floats = 512 MB at C3) -- format preparation, outside the step
    p_spmm = row_block(eng, p_dev, shard) if shard is not None else p_dev
    p_spmm = eng.block_columns(p_spmm, eng.panel_cols_for(p_spmm.shape[1], v_dev.shape[1]))
    p_block = p_spmm if shard is not None else None

    def mark(name):
        if phases is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            phases.append((name, ev))

    def step():
        mark("start")
        if shard is None:
            e = eng.spmm(p_spmm, v_dev, ell=v_dev.shape[1])
            mark("spmm")
            ids = eng.score_topk(e, v_dev, rank_r, topk, seen=seen)
            mark("fused_score_topk")
            return ids
        e = gather_embeddings(eng, p_block, v_dev, shard, n_users)
        mark("spmm_rows+allgather")
        v_slice = v_dev[shard.item_lo:shard.item_hi]
        chunk = shard.user_chunk(n_users)
        cands = eng.score_topk_cands(e, v_slice, rank_r, topk, seen=seen, item_offset=shard.item_lo, m=n_users,
                                     m_alloc=chunk * shard.world, bound_max=max_over_ranks if shard.world > 1 else None)
        mark("fused_score_topk")
        recv = exchange_candidates(cands, shard.world)
        mark("exchange")
        ids = merge_owned(eng, recv, e, v_dev, rank_r, topk, seen, shard, n_users)
        mark("merge")
        return ids
    return step


def time_score_kernel(eng, p_dev, v_dev, rank_r, topk, shard=None, reps=3):
    """Average duration (ms) of the fused scoring kernel alone, read from the CUDA events the
    library records around that launch on the context stream."""
    e = eng.spmm(p_dev, v_dev, ell=v_dev.shape[1])
    seen = (p_dev.indptr, p_dev.indices)
    v_use = v_dev if shard is None else v_dev[shard.item_lo:shard.item_hi]
    off = 0 if shard is None else shard.item_lo
    total = 0.0
    for i in range(reps + 1):
        eng.score_topk(e, v_use, rank_r, topk, seen=seen, item_offset=off)
        ms = eng.last_score_kernel_ms()
        if i > 0:
            total += ms
    return total / reps


def make_e2e(model, shard=None):
    """The user-facing call: host CSR in, host recommendations out."""
    if shard is None:
        return model.get_recommendations
    model.shard = shard
    return model.get_recommendations

"""Host-side logic of the item-sharded path on CPU: shard bounds, user chunks and the candidate exchange
(gloo, world size 2).  The merge itself is a CUDA kernel and is covered by the GPU tests."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from polara_b200.dist import ItemShard, exchange_candidates


def test_item_shard_bounds_cover_everything():
    for world, n in ((2, 100_001), (4, 10), (8, 1_000_000), (3, 7)):
        shards = [ItemShard(r, world, n) for r in range(world)]
        assert shards[0].item_lo == 0 and shards[-1].item_hi == n
        for a, b in zip(shards[:-1], shards[1:]):
            assert a.item_hi == b.item_lo
        n_users = 1003
        chunk = shards[0].user_chunk(n_users)
        assert chunk * world >= n_users
        covered = sum(s.user_range(n_users)[1] - s.user_range(n_users)[0] for s in shards)
        assert covered == n_users


def test_item_shard_never_empty_and_refuses_more_ranks_than_items():
    for world, n in ((8, 13), (8, 8), (3, 4), (7, 100), (1, 2)):
        shards = [ItemShard(r, world, n) for r in range(world)]
        assert all(s.item_hi > s.item_lo for s in shards)
        assert max(s.item_hi - s.item_lo for s in shards) - min(s.item_hi - s.item_lo for s in shards) <= 1
    with pytest.raises(ValueError):
        ItemShard(0, 8, 7)


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, m_pad, k, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        # rank r's list entry for (user u, slot j) encodes (r, u, j) so the exchanged layout can be checked
        u = torch.arange(m_pad).view(m_pad, 1, 1)
        j = torch.arange(k).view(1, k, 1)
        cands = torch.cat([(rank * 1_000_000 + u * 100 + j).expand(m_pad, k, 1),
                           (-(rank * 1_000_000 + u * 100 + j)).expand(m_pad, k, 1)], dim=2).to(torch.int32).contiguous()
        recv = exchange_candidates(cands, world)
        np.save(os.path.join(out_dir, "recv%d.npy" % rank), recv.numpy())
    finally:
        dist.destroy_process_group()


def test_exchange_candidates_gloo_world2(tmp_path):
    world, m_pad, k = 2, 8, 3
    port = _free_port()
    mp.spawn(_worker, args=(world, port, m_pad, k, str(tmp_path)), nprocs=world, join=True)
    chunk = m_pad // world
    for rank in range(world):
        recv = np.load(tmp_path / ("recv%d.npy" % rank))
        assert recv.shape == (world, chunk, k, 2)
        for src in range(world):
            for lu in range(chunk):
                for j in range(k):
                    u = rank * chunk + lu          # rank owns users [rank*chunk, (rank+1)*chunk)
                    assert recv[src, lu, j, 0] == src * 1_000_000 + u * 100 + j
                    assert recv[src, lu, j, 1] == -(src * 1_000_000 + u * 100 + j)


# ----------------------------------------------------------------------------------------------------------------
# Row-sharded build (SURVEY.md 8e "Partitioning - build"): the CUDA library sums three things over the row shards
# through its reduce hook -- the Gram matrix of the user-side panel, the item-side panel A^T W and (ScaledSVD) the
# column counts.  The restatement below runs exactly that schedule on CPU tensors with gloo and must land on the
# singular values of the whole matrix.

def _svqb(y, reduce=None):
    g = y.T @ y
    if reduce is not None:
        reduce(g)
    lam, vec = torch.linalg.eigh(g)
    lam, vec = lam.flip(0), vec.flip(1)
    return y @ (vec * lam.clamp_min(1e-300).rsqrt()), lam


def _sharded_build_worker(rank, world, port, out_dir):
    from polara_b200.models import csr_row_block
    import scipy.sparse as sps
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rng = np.random.default_rng(11)
        m, n, r, ell = 301, 120, 6, 32
        dense = (rng.standard_normal((m, 8)) * 0.7 ** np.arange(8)) @ rng.standard_normal((8, n))
        dense[rng.random((m, n)) < 0.6] = 0.0
        a = sps.csr_matrix(dense)
        shard = ItemShard(rank, world, n)
        lo, hi = shard.user_range(m)
        ip, ix, vl, shp = csr_row_block(a.indptr, a.indices, a.data, a.shape, lo, hi)
        a_g = torch.from_numpy(sps.csr_matrix((vl, ix, ip), shape=shp).toarray())
        q = torch.from_numpy(np.random.default_rng(1).standard_normal((n, ell)))
        for _ in range(10):
            w, _ = _svqb(a_g @ q, dist.all_reduce)            # user-side panel: Gram summed over the shards
            z = a_g.T @ w
            dist.all_reduce(z)                                 # A^T W = sum_g A_g^T W_g
            q, _ = _svqb(z)                                    # item side: redundant on every rank
        b = a_g @ q
        g = b.T @ b
        dist.all_reduce(g)
        lam = torch.linalg.eigvalsh(g).flip(0)
        np.save(os.path.join(out_dir, "sigma%d.npy" % rank), lam[:r].clamp_min(0).sqrt().numpy())
        counts = torch.from_numpy(np.bincount(ix, minlength=n))
        dist.all_reduce(counts)                                # ScaledSVD column counts are global
        np.save(os.path.join(out_dir, "counts%d.npy" % rank), counts.numpy())
        if rank == 0:
            np.save(os.path.join(out_dir, "truth.npy"), np.linalg.svd(dense, compute_uv=False)[:r])
            np.save(os.path.join(out_dir, "truth_counts.npy"), a.getnnz(axis=0))
    finally:
        dist.destroy_process_group()


def test_row_sharded_build_schedule_gloo_world2(tmp_path):
    world = 2
    mp.spawn(_sharded_build_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    truth = np.load(tmp_path / "truth.npy")
    for rank in range(world):
        np.testing.assert_allclose(np.load(tmp_path / ("sigma%d.npy" % rank)), truth, rtol=1e-8)
        np.testing.assert_array_equal(np.load(tmp_path / ("counts%d.npy" % rank)), np.load(tmp_path / "truth_counts.npy"))
    np.testing.assert_array_equal(np.load(tmp_path / "sigma0.npy"), np.load(tmp_path / "sigma1.npy"))


def test_csr_row_block_views():
    from polara_b200.models import csr_row_block
    import scipy.sparse as sps
    a = sps.random(50, 20, density=0.2, random_state=3, format="csr")
    for lo, hi in ((0, 50), (0, 0), (7, 31), (49, 50)):
        ip, ix, vl, shp = csr_row_block(a.indptr, a.indices, a.data, a.shape, lo, hi)
        got = sps.csr_matrix((vl, ix, ip), shape=shp)
        assert (got != a[lo:hi]).nnz == 0
        tip, tix, tvl, _ = csr_row_block(torch.from_numpy(a.indptr.astype(np.int64)), torch.from_numpy(a.indices),
                                         torch.from_numpy(a.data), a.shape, lo, hi)
        assert np.array_equal(tip.numpy(), ip) and np.array_equal(tix.numpy(), ix) and np.array_equal(tvl.numpy(), vl)


def _gather_worker(rank, world, port, n_users, k, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from polara_b200.dist import gather_lists
        shard = ItemShard(rank, world, 1000)
        lo, hi = shard.user_range(n_users)
        mine = (np.arange(lo, hi)[:, None] * 100 + np.arange(k)[None, :]).astype(np.int64)     # row u holds u*100 + slot
        full = gather_lists(mine, shard, n_users, torch.device("cpu"))
        # the model does not know the user count of a test CSR that was handed over ready-made: it is the sum of the shares
        assert np.array_equal(gather_lists(mine, shard, None, torch.device("cpu")), full)
        np.save(os.path.join(out_dir, "full%d.npy" % rank), full)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("n_users", [1003, 8, 2])
def test_gather_lists_assembles_all_users_gloo_world2(tmp_path, n_users):
    """model.recommendations on an item-sharded model = the per-rank slices (users each rank owns) all-gathered into the
    full [n_users x k] array, identical on every rank, rows in user order, padding rows dropped."""
    world, k = 2, 4
    port = _free_port()
    mp.spawn(_gather_worker, args=(world, port, n_users, k, str(tmp_path)), nprocs=world, join=True)
    want = (np.arange(n_users)[:, None] * 100 + np.arange(k)[None, :]).astype(np.int64)
    for rank in range(world):
        np.testing.assert_array_equal(np.load(tmp_path / ("full%d.npy" % rank)), want)


def _bound_worker(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from polara_b200.dist import max_over_ranks
        # per-user lower bounds as two shards would hold them: -inf where a shard found fewer than k unseen probe items
        t = torch.tensor([1.0, -float("inf"), 3.0, -float("inf")]) if rank == 0 else torch.tensor([2.0, 0.5, -1.0, -float("inf")])
        max_over_ranks(t)
        np.save(os.path.join(out_dir, "bound%d.npy" % rank), t.numpy())
    finally:
        dist.destroy_process_group()


def test_bound_hook_takes_the_elementwise_maximum_gloo_world2(tmp_path):
    """the hook of item-sharded scoring (pb200_set_bound_hook): every rank ends up with the best bound any shard found;
    a user without a bound anywhere keeps -inf."""
    port = _free_port()
    mp.spawn(_bound_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    want = np.array([2.0, 0.5, 3.0, -np.inf], dtype=np.float32)
    for rank in range(2):
        np.testing.assert_array_equal(np.load(tmp_path / ("bound%d.npy" % rank)), want)


def test_both_sharded_scoring_call_sites_share_their_bounds():
    """sharded_topk (models) and make_step (bench) must hand the bound hook to score_topk_cands when more than one rank
    takes part -- a call site that forgets it still returns correct lists, only slower, so no parity test would notice."""
    import inspect
    from polara_b200 import dist as pdist
    for fn in (pdist.sharded_topk, pdist.make_step):
        src = inspect.getsource(fn)
        assert "score_topk_cands" in src and "bound_max=max_over_ranks if shard.world > 1 else None" in src, fn.__name__

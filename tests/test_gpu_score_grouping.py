"""Early termination of the tensor-core scoring sweep with users grouped by sweep length and the live cut
(csrc/topk_tc.cu, DESIGN.md 3.1): lists bit-equal to the exact SIMT kernel and to the full sweep, and the tile-product
counter (stats [5]) below what tiles formed by user index, or the probe bound alone, would execute."""
import numpy as np
import pytest
import torch

from tests.helpers import random_seen_csr

pytestmark = pytest.mark.gpu

BM = BN = 128          # users / items per tile
PROBE = 256            # largest-norm items scored exactly up front (two item tiles)


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    e = get_engine(0)
    yield e
    e.set_prune(True)
    e.set_score_kernel("tc")


def _upload(eng, e, v, indptr, cols):
    return eng.upload(e), eng.upload(v), (eng.upload(indptr), eng.upload(cols.astype(np.int32)))


def _score_all(eng, e_dev, v_dev, r, k, seen):
    """simt, tc full sweep, tc with early termination: (ids, scores, tile products executed, full)"""
    out = {}
    for name, kernel, prune in (("simt", "simt", True), ("full", "tc", False), ("cut", "tc", True)):
        eng.set_score_kernel(kernel)
        eng.set_prune(prune)
        s0 = eng.stats()
        ids, sc = eng.score_topk(e_dev, v_dev, r, k, seen=seen, want_scores=True)
        s1 = eng.stats()
        out[name] = (ids.cpu().numpy(), sc.cpu().numpy(), s1[5] - s0[5], s1[6] - s0[6])
    eng.set_prune(True)
    eng.set_score_kernel("tc")
    for name in ("full", "cut"):
        np.testing.assert_array_equal(out["simt"][0], out[name][0], err_msg=name)
        np.testing.assert_array_equal(out["simt"][1], out[name][1], err_msg=name)
    assert out["full"][2] == out["full"][3] > 0
    return out


def _host_needs(e, v, seen_rows, seen_cols, k):
    """Item tiles each user needs under the probe bound (first_cut_tile with t0 = k-th best unseen probe score), on the
    host in float64.  The norms are inflated a little more than the kernel's and t0 deflated, so these needs are never
    smaller than the kernel's."""
    m, n = e.shape[0], v.shape[0]
    item_tiles = -(-n // BN)
    vn = np.linalg.norm(v.astype(np.float64), axis=1)
    order = np.argsort(-vn, kind="stable")
    vn_sorted = vn[order] * 1.001
    en = np.linalg.norm(e.astype(np.float64), axis=1) * 1.001
    n_probe = min(PROBE, (n // BN) * BN)
    probe = order[:n_probe]
    s = e.astype(np.float64) @ v[probe].astype(np.float64).T
    slot = np.full(n, -1)
    slot[probe] = np.arange(n_probe)
    hit = slot[seen_cols] >= 0
    s[seen_rows[hit], slot[seen_cols[hit]]] = -np.inf
    t0 = -np.sort(-s, axis=1)[:, k - 1] if n_probe >= k else np.full(m, -np.inf)
    t0 = t0 - 1e-4 * np.abs(t0)
    starts = vn_sorted[np.arange(item_tiles) * BN]
    below = en[:, None] * starts[None, :] < t0[:, None]
    cut = np.isfinite(t0) & (t0 > 0) & below.any(axis=1)
    return np.where(cut, below.argmax(axis=1), item_tiles), n_probe // BN


def _tile_products(need, tile_first):
    """sum over 128-user tiles of the tile's sweep length (its largest need), for users taken in the given order"""
    total = 0
    for g in range(0, len(need), BM):
        total += max(int(need[g:g + BM].max()) - tile_first, 0)
    return total


def _skewed(rng, m, n, r):
    e = rng.standard_normal((m, r)).astype(np.float32)
    v = (rng.standard_normal((n, r)) * (1.0 / np.arange(1, n + 1) ** 0.8)[rng.permutation(n), None]).astype(np.float32)
    return e, v


def test_grouping_interleaved_sweep_lengths(eng):
    """Every odd user has seen the whole probe head (t0 = -inf: it needs the full sweep), the even ones have not.  Tiles
    formed by user index all contain odd users and sweep everything; grouped by need, half of the tiles are short."""
    rng = np.random.default_rng(101)
    m, n, r, k = 1000, 40000, 32, 10
    e, v = _skewed(rng, m, n, r)
    head = np.argsort(-np.linalg.norm(v.astype(np.float64), axis=1), kind="stable")[:PROBE + 64]
    per_row = rng.integers(0, 30, size=m)
    rows, cols, indptr = random_seen_csr(rng, m, n, per_row)
    # odd users: the probe head (and then some) on top of their random history
    r_l, c_l = [], []
    for u in range(m):
        c = cols[indptr[u]:indptr[u + 1]]
        if u % 2:
            c = np.union1d(c, head)
        r_l.append(np.full(len(c), u)); c_l.append(np.sort(c))
    rows, cols = np.concatenate(r_l), np.concatenate(c_l)
    indptr = np.zeros(m + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=m), out=indptr[1:])
    e_dev, v_dev, seen = _upload(eng, e, v, indptr, cols)
    out = _score_all(eng, e_dev, v_dev, r, k, seen)
    need, tile_first = _host_needs(e, v, rows, cols, k)
    assert (need[1::2] == -(-n // BN)).all()
    grouped = _tile_products(np.sort(need)[::-1], tile_first)
    by_index = _tile_products(need, tile_first)
    executed = out["cut"][2]
    assert executed <= grouped, (executed, grouped)
    assert executed < 0.7 * by_index, (executed, by_index)
    # run to run: same bits
    ids2, sc2 = eng.score_topk(e_dev, v_dev, r, k, seen=seen, want_scores=True)
    np.testing.assert_array_equal(ids2.cpu().numpy(), out["cut"][0])
    np.testing.assert_array_equal(sc2.cpu().numpy(), out["cut"][1])


def test_live_cut_stops_below_the_probe_bound(eng):
    """The 256 largest-norm items are nearly orthogonal to every user (t0 is tiny), strongly aligned items follow right
    behind them, then a tail of random items whose norms fall from 8.  Under t0 alone nearly the whole tail must be
    swept; once the aligned items are in the lists (scores ~ 9 ||e||) nothing in the tail can enter, and the sweep stops.
    The live bound grows inside a work item, so there are enough user tiles (2 per SM) for the sweep not to be split
    into item parts, each of which would start again from t0."""
    rng = np.random.default_rng(102)
    m, n, r, k = 34000, 20000, 32, 10
    n_head, n_aligned = PROBE, 1000
    d = np.zeros(r); d[0] = 1.0
    a = rng.uniform(0.5, 1.5, size=m)
    e = a[:, None] * d[None, :]
    e[:, 1:16] += 0.01 * rng.standard_normal((m, 15))                 # users live in the first 16 dimensions
    head = np.zeros((n_head, r))
    w = rng.standard_normal((n_head, 16))
    head[:, 16:] = 10.0 * w / np.linalg.norm(w, axis=1, keepdims=True)  # norm ~10, orthogonal to the users ...
    head[:, 0] = rng.uniform(0.04, 0.06, size=n_head)                   # ... but for a small positive score
    aligned = 9.0 * d[None, :] + np.concatenate([np.zeros((n_aligned, 1)), 0.05 * rng.standard_normal((n_aligned, 15)),
                                                 np.zeros((n_aligned, r - 16))], axis=1)
    n_tail = n - n_head - n_aligned
    t = rng.standard_normal((n_tail, r))
    tail = t / np.linalg.norm(t, axis=1, keepdims=True) * np.geomspace(8.0, 0.01, n_tail)[:, None]
    v = np.concatenate([head, aligned, tail])[rng.permutation(n)]
    e, v = e.astype(np.float32), v.astype(np.float32)
    rows, cols, indptr = random_seen_csr(rng, m, n, rng.integers(0, 8, size=m))
    e_dev, v_dev, seen = _upload(eng, e, v, indptr, cols)
    out = _score_all(eng, e_dev, v_dev, r, k, seen)
    need, tile_first = _host_needs(e, v, rows, cols, k)
    static = _tile_products(np.sort(need)[::-1], tile_first)
    executed = out["cut"][2]
    assert executed < 0.5 * static, (executed, static)


@pytest.mark.parametrize("m", [1000, 77, 129])
def test_grouping_partial_tiles(eng, m):
    """m not a multiple of 128, and m < 128 (one user tile, the sweep split into item parts)"""
    rng = np.random.default_rng(110 + m)
    n, r, k = 30000, 50, 10
    e, v = _skewed(rng, m, n, r)
    rows, cols, indptr = random_seen_csr(rng, m, n, rng.integers(0, 60, size=m))
    e_dev, v_dev, seen = _upload(eng, e, v, indptr, cols)
    out = _score_all(eng, e_dev, v_dev, r, k, seen)
    assert out["cut"][2] < out["cut"][3]


def test_grouping_all_negative_scores_cut_nothing(eng):
    rng = np.random.default_rng(120)
    m, n, r, k = 600, 20000, 50, 10
    e, v = _skewed(rng, m, n, r)
    v = -np.abs(v); e = np.abs(e)
    rows, cols, indptr = random_seen_csr(rng, m, n, rng.integers(0, 60, size=m))
    e_dev, v_dev, seen = _upload(eng, e, v, indptr, cols)
    out = _score_all(eng, e_dev, v_dev, r, k, seen)
    assert out["cut"][2] == out["cut"][3]


def test_grouping_zero_norm_item_tail(eng):
    rng = np.random.default_rng(130)
    m, n, r, k = 700, 30000, 50, 10
    e = rng.standard_normal((m, r)).astype(np.float32)
    v = (np.abs(rng.standard_normal((n, r))) * (1.0 / np.arange(1, n + 1) ** 0.8)[:, None]).astype(np.float32)
    v[n // 2:] = 0.0                                     # exact zeros score 0 ...
    e[: m // 2] = -np.abs(e[: m // 2])                   # ... and must beat these users' all-negative other scores
    rows, cols, indptr = random_seen_csr(rng, m, n, rng.integers(0, 60, size=m))
    e_dev, v_dev, seen = _upload(eng, e, v, indptr, cols)
    _score_all(eng, e_dev, v_dev, r, k, seen)


def test_grouping_k_above_32(eng):
    rng = np.random.default_rng(140)
    m, n, r, k = 500, 30000, 50, 40
    e, v = _skewed(rng, m, n, r)
    rows, cols, indptr = random_seen_csr(rng, m, n, rng.integers(0, 60, size=m))
    e_dev, v_dev, seen = _upload(eng, e, v, indptr, cols)
    out = _score_all(eng, e_dev, v_dev, r, k, seen)
    assert out["cut"][2] < out["cut"][3]


def test_grouping_sharded_with_bound_hook(eng):
    """item shards exchange their bounds through the hook (the need of every user is recomputed from the shared
    bound): merged lists equal the unsharded ones"""
    rng = np.random.default_rng(150)
    m, n, r, k = 700, 24000, 32, 10
    e = rng.standard_normal((m, r)).astype(np.float32)
    v = (rng.standard_normal((n, r)) * np.geomspace(4.0, 0.05, n)[:, None]).astype(np.float32)
    rows, cols, indptr = random_seen_csr(rng, m, n, rng.integers(0, 60, size=m))
    e_dev, v_dev, seen = _upload(eng, e, v, indptr, cols)
    eng.set_score_kernel("simt")
    ref = eng.score_topk(e_dev, v_dev, r, k, seen=seen).cpu().numpy()
    eng.set_score_kernel("tc")
    bounds = [0, 8000, 16000, 24000]
    shards = [(lo, eng.upload(v[lo:hi])) for lo, hi in zip(bounds[:-1], bounds[1:])]
    own = []
    for lo, v_s in shards:
        eng.score_topk_cands(e_dev, v_s, r, k, seen=seen, item_offset=lo, bound_max=lambda t: own.append(t.clone()))
    best = torch.stack(own).max(dim=0).values
    parts = [eng.score_topk_cands(e_dev, v_s, r, k, seen=seen, item_offset=lo, bound_max=lambda t: t.copy_(best))
             for lo, v_s in shards]
    merged = eng.merge_cands(torch.stack(parts).contiguous(), len(parts), m, k).cpu().numpy()
    np.testing.assert_array_equal(merged, ref)

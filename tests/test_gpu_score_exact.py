"""The scoring kernels bit for bit against the host emulation of their contract (tests/exact_scoring.py, DESIGN.md §3.1
and §4 "Scoring"): every reported score is the canonical fp32 chain, every list is the k best under (score desc, id asc)
with -0 == +0, unseen items first and the seen ones after them.  Ids and score bits are compared, no tolerance.

pb200_score_topk runs three ways (CUDA-core SIMT kernel; tensor-core kernel with and without the early termination), the
item-sharded path is emulated in one process down to the real merge of dist.merge_owned, and pb200_score_dense,
pb200_gather_dot and pb200_topk_dense are checked on their own.  The inputs aim at ties (small integer factors,
duplicated items, zero rows, a k-th best score of exactly 0), signed zeros (products that underflow), extreme scales,
the K boundaries of the tensor-core operands, unaligned column-slice views with NaN beyond column r, tile edges in n and
m, and k from 1 to 1024 and beyond n.  H100 only."""
import numpy as np
import pytest
import torch

from tests.exact_scoring import canonical_scores, csr_of, expected_cands, expected_lists

pytestmark = pytest.mark.gpu

KERNELS = ("simt", "tc_cut", "tc_full")


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    e = get_engine(0)
    yield e
    e.set_score_kernel("tc")
    e.set_prune(True)


def _set_kernel(eng, kernel):
    eng.set_score_kernel("simt" if kernel == "simt" else "tc")
    eng.set_prune(kernel != "tc_full")


def _on_device(eng, X, r, layout):
    """X [rows x r] float32 as the kernels see it: ``aligned`` = padded to 32 columns (16-byte rows, the engine's own
    layout, vector loads); ``odd`` = a column-slice view at column 1 of a buffer with an odd leading dimension (scalar
    loads).  Every column outside [0, r) holds NaN."""
    rows = X.shape[0]
    if layout == "aligned":
        buf = np.full((rows, -(-r // 32) * 32), np.nan, np.float32)
        buf[:, :r] = X[:, :r]
        return eng.upload(buf)
    ld = r + 2 + (r + 1) % 2                               # odd, >= r + 2
    buf = np.full((rows, ld), np.nan, np.float32)
    buf[:, 1:1 + r] = X[:, :r]
    view = eng.upload(buf)[:, 1:1 + r]
    assert view.stride(0) % 2 == 1 and view.data_ptr() % 16 != 0
    return view


def _seen_dev(eng, seen):
    return None if seen is None else (eng.upload(seen[0]), eng.upload(seen[1]))


def _assert_same(label, ids, scores, exp_ids, exp_scores):
    """ids equal and score bits equal; on a mismatch the message names the rows that differ"""
    ids = np.asarray(ids, np.int64)
    sb = np.asarray(scores, np.float32).view(np.uint32)
    eb = np.asarray(exp_scores, np.float32).view(np.uint32)
    bad = np.flatnonzero(((ids != exp_ids) | (sb != eb)).any(axis=1))
    if len(bad):
        u = bad[0]
        j = np.flatnonzero((ids[u] != exp_ids[u]) | (sb[u] != eb[u]))[:6]
        raise AssertionError("%s: %d rows differ (first %s); row %d at %s: got ids %s scores %s, expected ids %s scores %s"
                             % (label, len(bad), bad[:10].tolist(), u, j.tolist(), ids[u, j].tolist(),
                                np.asarray(scores)[u, j].tolist(), exp_ids[u, j].tolist(),
                                np.asarray(exp_scores)[u, j].tolist()))


def _check_score_topk(eng, E, V, r, k, seen=None, item_offset=0, layout="aligned", kernels=KERNELS):
    S = canonical_scores(E, V, r)
    exp_ids, exp_sc = expected_lists(S, seen, k, item_offset)
    e_dev, v_dev = _on_device(eng, E, r, layout), _on_device(eng, V, r, layout)
    sd = _seen_dev(eng, seen)
    try:
        for kernel in kernels:
            _set_kernel(eng, kernel)
            ids, sc = eng.score_topk(e_dev, v_dev, r, k, seen=sd, item_offset=item_offset, want_scores=True)
            _assert_same(kernel, ids.cpu().numpy(), sc.cpu().numpy(), exp_ids, exp_sc)
    finally:
        _set_kernel(eng, "tc_cut")
    return S


def _head(V, r, count=300):
    """the largest-norm items (a superset of the tensor-core probe's 256-item head)"""
    return np.argsort(-np.linalg.norm(V[:, :r].astype(np.float64), axis=1), kind="stable")[:count]


# ------------------------------------------------------------------------------------------------------------------------
#  shapes: K boundaries of the tensor-core operands (61/62 one slab, 64/65 the K atom), tile edges, k up to 1024 and > n
# ------------------------------------------------------------------------------------------------------------------------
SHAPES = [  # m, n, r, k, layout, seen, item_offset
    (63, 257, 1, 1, "aligned", "none", 0),
    (65, 255, 3, 32, "odd", "random", 0),
    (129, 256, 31, 33, "aligned", "head", 0),
    (129, 1025, 61, 256, "aligned", "random", 0),
    (65, 1023, 62, 300, "odd", "none", 0),
    (1, 1, 63, 32, "aligned", "none", 0),
    (129, 2049, 64, 1024, "aligned", "head", 0),
    (63, 1025, 65, 33, "odd", "all_but_few", 0),
    (129, 767, 129, 32, "aligned", "random", 1000),
    (33, 300, 129, 300, "odd", "all_but_few", 7),
]


def _seen_for(kind, rng, m, n, V, r, k, offset):
    if kind == "none":
        return None
    if kind == "head":                                     # covers the whole probe head (and some more) for half the users
        h = _head(V, r)
        return csr_of([h + offset if u % 2 == 0 else rng.choice(n, 5, replace=False) + offset for u in range(m)], m)
    if kind == "all_but_few":                              # fewer than k unseen items (none for some users)
        rows = []
        for u in range(m):
            keep = rng.choice(n, size=min(n, u % (k + 1)), replace=False)
            rows.append(np.setdiff1d(np.arange(n), keep) + offset)
        return csr_of(rows, m)
    return csr_of([rng.choice(n, size=rng.integers(0, min(n, 60) + 1), replace=False) + offset for _ in range(m)], m)


@pytest.mark.parametrize("m,n,r,k,layout,seen_kind,offset", SHAPES,
                         ids=["m%d-n%d-r%d-k%d-%s-%s-off%d" % s for s in SHAPES])
def test_score_topk_shapes(eng, m, n, r, k, layout, seen_kind, offset):
    rng = np.random.default_rng(m * 7919 + n * 31 + r)
    E = rng.standard_normal((m, r)).astype(np.float32)
    V = rng.standard_normal((n, r)).astype(np.float32)
    if n > 20:
        V[n // 2: n // 2 + 5] = V[3:8]                      # duplicated items: exact ties decided by the id
    seen = _seen_for(seen_kind, rng, m, n, V, r, k, offset)
    _check_score_topk(eng, E, V, r, k, seen, offset, layout)


# ------------------------------------------------------------------------------------------------------------------------
#  ties
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 10, 33, 256])
def test_score_topk_massive_ties(eng, k):
    """factors in {-2..2}: most scores tie and the id decides.  Duplicated item rows inside and outside the probe head,
    zero user rows, random seen lists."""
    rng = np.random.default_rng(11 + k)
    m, n, r = 200, 1500, 8
    E = rng.integers(-2, 3, (m, r)).astype(np.float32)
    V = rng.integers(-2, 3, (n, r)).astype(np.float32)
    E[::17] = 0.0
    head = _head(V, r, 256)
    V[[1, 2, 3]] = V[head[:3]]                             # a low-id copy of head items
    V[[1400, 1401]] = V[head[3:5]]                         # a high-id copy of head items
    V[[40, 41, 900]] = V[50]                               # copies outside the head
    seen = csr_of([rng.choice(n, size=rng.integers(0, 40), replace=False) for _ in range(m)], m)
    _check_score_topk(eng, E, V, r, k, seen)
    _check_score_topk(eng, E, V, r, k, None)


@pytest.mark.parametrize("k", [1, 10, 33])
def test_score_topk_kth_score_exactly_zero(eng, k):
    """A k-th best score of exactly 0 with zero-norm items of low id: they tie with the probe's winners and must enter
    by their id.  User 0 has an all-zero row; user 1 scores exactly 0 on every item outside its two columns (disjoint
    supports), with fewer than k items above 0 and at least k head items at 0; user 2 is user 0 with items 0..4 seen."""
    rng = np.random.default_rng(5 + k)
    m, n, r = 70, 1000, 8
    V = rng.integers(-2, 3, (n, r)).astype(np.float32)
    V[:, :2] = 0.0                                         # every item lives on columns 2..7 ...
    pos = rng.choice(np.arange(300, n), size=k // 2, replace=False)
    V[pos, 0] = 1.0                                        # ... except fewer than k that score > 0 for user 1
    V[rng.choice(np.arange(300, n), size=5, replace=False), 1] = -1.0
    V[:20] = 0.0                                           # zero-norm items with the lowest ids
    E = rng.integers(-2, 3, (m, r)).astype(np.float32)
    E[0] = 0.0
    E[1] = 0.0
    E[1, :2] = [1.0, 2.0]
    E[2] = 0.0
    seen = csr_of([[], [], np.arange(5)] + [rng.choice(n, size=10, replace=False) for _ in range(m - 3)], m)
    S = _check_score_topk(eng, E, V, r, k, seen)
    assert np.sort(S[1])[::-1][k - 1] == 0.0 and (S[1, _head(V, r, 256)] == 0).sum() >= k


@pytest.mark.parametrize("n", [256, 1000])
@pytest.mark.parametrize("k", [10, 33])
def test_score_topk_signed_zero_scores(eng, n, k):
    """Factors near 2^-77: every product underflows, so every score is +0 or -0 (a chain ends at -0 when its last nonzero
    product was negative).  The two zeros tie and the id decides, in the probe's head as well as in the sweep; the
    reported score keeps the chain's sign."""
    rng = np.random.default_rng(n + k)
    m, r = 64, 8
    E = (rng.integers(-2, 3, (m, r)) * 2.0 ** -77).astype(np.float32)
    V = (rng.integers(-2, 3, (n, r)) * 2.0 ** -77).astype(np.float32)
    S = _check_score_topk(eng, E, V, r, k)
    assert np.all(S == 0) and np.signbit(S).any() and (~np.signbit(S)).any()


# ------------------------------------------------------------------------------------------------------------------------
#  scale
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["per_user", "tiny", "huge", "subnormal"])
def test_score_topk_scales(eng, case):
    """per-user scales 2^-40 .. 2^40 inside one 128-user tile; whole problems at 2^-60 and 2^60 (scores stay finite);
    subnormal factor entries (and subnormal scores)"""
    rng = np.random.default_rng({"per_user": 1, "tiny": 2, "huge": 3, "subnormal": 4}[case])
    m, n, r, k = 128, 1100, 24, 20
    E = rng.standard_normal((m, r)).astype(np.float32)
    V = rng.standard_normal((n, r)).astype(np.float32)
    if case == "per_user":
        E *= np.exp2(np.round(np.linspace(-40, 40, m)))[:, None].astype(np.float32)
    elif case == "tiny":
        E *= np.float32(2.0 ** -60)
        V *= np.float32(2.0 ** -60)
    elif case == "huge":
        E *= np.float32(2.0 ** 60)
        V *= np.float32(2.0 ** 58)
    else:
        E[: m // 2] *= np.float32(2.0 ** -130)              # subnormal user rows: subnormal scores
        V[::3] *= np.float32(2.0 ** -20)
        V[5::7, :4] = np.float32(2.0 ** -140)
    seen = csr_of([rng.choice(n, size=rng.integers(0, 30), replace=False) for _ in range(m)], m)
    S = _check_score_topk(eng, E, V, r, k, seen)
    assert np.isfinite(S).all()


# ------------------------------------------------------------------------------------------------------------------------
#  score_dense, gather_dot
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [1, 33, 100])
@pytest.mark.parametrize("r,layout", [(1, "aligned"), (33, "odd"), (64, "aligned"), (129, "odd")])
def test_score_dense_and_gather_dot_are_canonical(eng, m, r, layout):
    rng = np.random.default_rng(m * 1000 + r)
    n = 999
    E = rng.standard_normal((m, r)).astype(np.float32)
    V = rng.standard_normal((n, r)).astype(np.float32)
    E[0, : r // 2] *= np.float32(2.0 ** -75)               # underflowing products and signed zeros in the first row
    V[: n // 3] *= np.float32(2.0 ** -75)
    S = canonical_scores(E, V, r)
    e_dev, v_dev = _on_device(eng, E, r, layout), _on_device(eng, V, r, layout)
    got = eng.score_dense(e_dev, v_dev, r).cpu().numpy()
    np.testing.assert_array_equal(got.view(np.uint32), S.view(np.uint32))
    u = rng.integers(-1, m + 1, 5000)
    j = rng.integers(-1, n + 1, 5000)
    u[:3], j[:3] = [0, m, -1], [n, 0, 0]
    out = eng.gather_dot(e_dev, v_dev, r, eng.upload(u), eng.upload(j)).cpu().numpy()
    ok = (u >= 0) & (u < m) & (j >= 0) & (j < n)
    assert np.isnan(out[~ok]).all() and (~ok).sum() >= 3
    np.testing.assert_array_equal(out[ok].view(np.uint32), S[u[ok], j[ok]].view(np.uint32))


# ------------------------------------------------------------------------------------------------------------------------
#  topk_dense
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n,k", [(300, 10), (300, 33), (77, 77), (1, 1), (2000, 256)])
def test_topk_dense_ties_zeros_and_fill(eng, dtype, n, k):
    """massive exact ties (values in {-2..2}), +-0, -inf and NaN entries, a seen CSR that leaves fewer than k unseen items
    (or none), k = n"""
    rng = np.random.default_rng(n + k)
    m = 70
    S = rng.integers(-2, 3, (m, n)).astype(dtype)
    zero = rng.random((m, n)) < 0.3
    S[zero] = np.where(rng.random(zero.sum()) < 0.5, 0.0, -0.0)
    S[rng.random((m, n)) < 0.05] = -np.inf
    S[rng.random((m, n)) < 0.02] = np.nan
    S[1] = -0.0
    S[2] = -np.inf
    rows = []
    for u in range(m):
        if u % 3 == 0:                                     # fewer than k unseen (none for some)
            rows.append(np.setdiff1d(np.arange(n), rng.choice(n, size=min(n, u % (k + 1)), replace=False)))
        else:
            rows.append(rng.choice(n, size=rng.integers(0, n // 2 + 1), replace=False))
    seen = csr_of(rows, m)
    s_dev = eng.upload(S)
    for sd in (seen, None):
        exp_ids, exp_sc = expected_lists(S, sd, k)
        ids, sc = eng.topk_dense(s_dev, k, seen=_seen_dev(eng, sd), want_scores=True)
        ids, sc = ids.cpu().numpy(), sc.cpu().numpy()
        np.testing.assert_array_equal(ids, exp_ids)
        view = np.uint64 if dtype == np.float64 else np.uint32
        np.testing.assert_array_equal(sc.view(view), exp_sc.view(view))
    with pytest.raises(Exception):
        eng.topk_dense(s_dev, n + 1)                       # k > n is refused (np.argpartition raises too)


# ------------------------------------------------------------------------------------------------------------------------
#  the item-sharded path, emulated in one process
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world,n", [(2, 600), (3, 1000), (8, 13), (8, 700)])
@pytest.mark.parametrize("kernel", ["simt", "tc_cut"])
def test_sharded_candidates_and_merge(eng, world, n, kernel):
    """ItemShard ranges, score_topk_cands per shard (user rows padded to world x chunk), the exchange layout built by
    slicing as exchange_candidates returns it, then the real dist.merge_owned: merge_cands_fill with part_stride =
    chunk x k and fewer than chunk owned users on the last rank, and merge_cands without seen lists.  Users with fewer than
    k unseen items over all shards, users with none, shards smaller than k."""
    from polara_b200 import dist
    rng = np.random.default_rng(world * 100 + n)
    m, r, k = 71, 16, 10
    E = rng.integers(-2, 3, (m, r)).astype(np.float32)
    V = rng.integers(-2, 3, (n, r)).astype(np.float32)
    E[0] = 0.0
    rows = []
    for u in range(m):
        if u % 4 == 1:
            rows.append(np.setdiff1d(np.arange(n), rng.choice(n, size=min(n, u % (k + 1)), replace=False)))
        elif u % 4 == 2:
            rows.append(np.arange(n) if u % 8 == 2 else np.arange(0, n, 2))
        else:
            rows.append(rng.choice(n, size=min(n, rng.integers(0, 30)), replace=False))
    seen = csr_of(rows, m)
    S = canonical_scores(E, V, r)
    shards = [dist.ItemShard(w, world, n) for w in range(world)]
    assert all(s.item_hi > s.item_lo for s in shards) and shards[-1].item_hi == n
    chunk = shards[0].user_chunk(m)
    m_pad = chunk * world
    assert m - (world - 1) * chunk < chunk                 # the last rank owns fewer users than a chunk
    e_dev, v_dev = eng.upload(E), eng.upload(V)
    seen_dev = _seen_dev(eng, seen)
    _set_kernel(eng, kernel)
    try:
        for sd, sh in ((seen_dev, seen), (None, None)):
            cands = []
            for s in shards:
                c = eng.score_topk_cands(e_dev, v_dev[s.item_lo:s.item_hi], r, k, seen=sd, item_offset=s.item_lo, m=m,
                                         m_alloc=m_pad)
                exp_ids, exp_sc = expected_cands(S[:, s.item_lo:s.item_hi], sh, k, s.item_lo)
                got = c.cpu().numpy()
                _assert_same("shard %d cands" % s.rank, got[:m, :, 1], got[:m, :, 0].view(np.float32), exp_ids, exp_sc)
                assert (got[m:, :, 1] == -1).all() and (got[m:, :, 0].view(np.float32) == -np.inf).all()
                cands.append(c)
            exp_ids, _ = expected_lists(S, sh, k)
            for s in shards:
                lo, hi = s.user_range(m)
                recv = torch.stack([c[s.rank * chunk:(s.rank + 1) * chunk] for c in cands]).contiguous()
                ids = dist.merge_owned(eng, recv, e_dev, v_dev, r, k, sd, s, m).cpu().numpy()
                np.testing.assert_array_equal(ids[:hi - lo], exp_ids[lo:hi], err_msg="rank %d, seen=%s" % (s.rank, sd is not None))
                if sd is None:
                    assert (ids[hi - lo:] == -1).all()     # padding users: empty lists
    finally:
        _set_kernel(eng, "tc_cut")


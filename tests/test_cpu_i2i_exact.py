"""The host emulation of the item-to-item summation order (tests/i2i_exact.py) against scipy, and its fixtures against
what they promise.  CPU only: the GPU tests compare the kernels with this emulation bit for bit, so it has to equal
the reference's arithmetic, and its fixtures have to tell the order apart, first."""
import numpy as np
import pytest

from oracle import i2i_oracle as io
from oracle import sim_oracle as so
from tests import i2i_exact as ie


def _cooc_matrix(a):
    coo = a.tocoo()
    return io.cooc_matrix(np.c_[coo.row, coo.col], coo.data, a.shape)


def _bits_equal(x, y):
    return x.dtype == y.dtype and x.shape == y.shape and np.ascontiguousarray(x).tobytes() == \
        np.ascontiguousarray(y).tobytes()


def test_build_s_equals_scipy():
    """S = AᵀA, setdiag(0), eliminate_zeros() (oracle/i2i_oracle.cooc_matrix), dense and as a CSR"""
    c = ie.cooc_case()
    want = _cooc_matrix(c["a"])
    assert _bits_equal(c["s"], want.toarray())
    want.sort_indices()
    assert _bits_equal(c["s_csr"].indptr.astype(np.int64), want.indptr.astype(np.int64))
    assert _bits_equal(c["s_csr"].indices.astype(np.int64), want.indices.astype(np.int64))
    assert _bits_equal(c["s_csr"].data, want.data)
    w = ie.wide_case()
    assert _bits_equal(w["s"], _cooc_matrix(w["a"])[w["rows"]].toarray())


def test_build_s_equals_scipy_with_implicit():
    a = ie.cooc_case()["a"]
    coo = a.tocoo()
    want = io.cooc_matrix(np.c_[coo.row, coo.col], coo.data, a.shape, implicit=True).toarray()
    assert _bits_equal(ie.build_s(a, implicit=True), want)


def test_scores_equal_scipy():
    """P·S (oracle/i2i_oracle.scores) and P·M on SimilarityAggregation's operand, Sᵀ and S"""
    c = ie.cooc_case()
    assert _bits_equal(c["scores"], io.scores(c["p"], _cooc_matrix(c["a"])).toarray())
    for dense_output in (False, True):
        s = ie.sim_case(dense_output)
        want = io.scores(s["p"], so.scoring_operand(so.similarity_matrix(s["rel"]), dense_output)).toarray()
        assert _bits_equal(s["scores"], want)


def _stats(mask):
    return int(mask.sum())


def test_the_build_fixtures_tell_the_order_apart():
    """Summing the users in reverse changes the bits of at least this many entries: in table-path rows, in long-path
    rows, in each column panel of 100 and of 1000 columns, and in both panels of the full 8192-column width."""
    c = ie.cooc_case()
    d = ie.differs(c["s"], ie.build_s(c["a"], order="desc"))
    work = ie.build_work(c["a"])
    table, long_ = (work > 0) & (work <= ie.HASH_WORK), work > ie.HASH_WORK
    assert _stats(d[table]) >= 1000 and _stats(d[table].any(axis=1)) >= 200
    assert _stats(d[long_]) >= 3000 and _stats(d[long_].any(axis=1)) >= 50
    for width, least in ((100, 200), (1000, 1000)):
        for c0 in range(0, ie.COOC_ITEMS, width):
            assert _stats(d[:, c0:c0 + width]) >= least, (width, c0)
    for key in ("work", "raters"):
        for row in c["roles"][key].values():
            assert _stats(d[row]) >= 10, (key, row)
    w = ie.wide_case()
    dw = ie.differs(w["s"], ie.build_s(w["a"], order="desc", rows=w["rows"]))
    assert _stats(dw[:, :8192]) >= 2000 and _stats(dw[:, 8192:]) >= 50


@pytest.mark.parametrize("case", ["cooc", "sim", "sim_dense_output"])
def test_the_scoring_fixtures_tell_the_order_apart(case):
    """Summing a user's items in reverse changes the bits of at least this many scores, on both accumulator paths and
    for the users of work exactly 512 and 513."""
    if case == "cooc":
        c, mat = ie.cooc_case(), ie.cooc_case()["s_csr"]
    else:
        c = ie.sim_case(case == "sim_dense_output")
        mat = c["mat"]
    d = ie.differs(c["scores"], ie.scores(c["p"], mat, order="desc"))
    users = c["users"]
    assert _stats(d[users["heavy"]]) >= 5000
    assert _stats(d[users["light"]]) >= 500
    for target, u in users["work"].items():
        assert _stats(d[u]) >= 5, target


def test_the_cooc_fixture_has_its_structure():
    c = ie.cooc_case()
    for a in (c["a"], ie.wide_case()["a"]):
        v = a.data
        assert _bits_equal(v.astype(np.float32).astype(np.float64), v)             # fp32-representable
        assert (np.abs(v) < 2.0 ** -18).any() and (np.abs(v) >= 2.0 ** 19).any()   # exponents over 2⁻²⁰..2²⁰
        assert (v < 0).mean() > 0.4 and (v > 0).mean() > 0.4
        assert (np.ldexp(np.frexp(v)[0], 24) % 2 == 1).mean() > 0.4                 # full 24-bit mantissas
    a, roles, s = c["a"], c["roles"], c["s"]
    work = ie.build_work(a)
    raters = np.diff(a.tocsc().indptr)
    assert {t: int(work[i]) for t, i in roles["work"].items()} == {512: 512, 513: 513}
    assert {t: int(raters[i]) for t, i in roles["raters"].items()} == {128: 128, 129: 129, 257: 257}
    assert np.diff(a.indptr).max() > 2 * ie.BUILD_BATCH                   # more than two items per build thread
    assert (work > ie.HASH_WORK).sum() >= 10 and ((work > 0) & (work <= ie.HASH_WORK)).sum() >= 100
    pattern = a.copy()
    pattern.data[:] = 1.0
    co = (pattern.T @ pattern).toarray()
    for i, j in roles["cancel"]:
        assert co[i, j] == 2 and s[i, j] == 0 and s[j, i] == 0                # co-rated, summed to exactly 0
        assert s[i, j].view(np.int64) == 0 and s[j, i].view(np.int64) == 0   # +0
    assert ((co >= 3) & (s != 0)).sum() > 0.5 * (co >= 3).sum() and (co >= 3).sum() > 20000
    for x, y in roles["dup"]:
        keep = np.setdiff1d(np.arange(s.shape[1]), [x, y])
        assert _bits_equal(s[x, keep], s[y, keep]) and s[x, keep].any()


def test_the_test_users_have_their_structure():
    """both accumulator paths, work exactly 512 and 513, more than 32 items, cancellations to exactly 0 among touched
    columns on both paths, ties between duplicated columns inside the lists, zero feedback and an empty user"""
    c = ie.cooc_case()
    users, sc, p, s_csr = c["users"], c["scores"], c["p"], c["s_csr"]
    work = ie.score_work(p, s_csr)
    assert (work[users["heavy"]] > ie.HASH_WORK).all() and (work[users["light"]] <= ie.HASH_WORK).all()
    assert {t: int(work[u]) for t, u in users["work"].items()} == {512: 512, 513: 513}
    lens = np.diff(p.indptr)
    assert ((lens > ie.SCORE_BATCH) & (work > ie.HASH_WORK)).sum() >= 3
    assert lens[-1] == 0 and lens[-2] == 0 and np.diff(c["seen"].indptr)[-2] == 2
    assert (c["triplets"][2] == 0).sum() > 2 + 5                           # zero feedback beyond the seen-only user
    assert ie.COOC_ITEMS % ie.SCORE_PANEL and ie.COOC_ITEMS > 4 * ie.SCORE_PANEL
    pattern, s_pat = p.copy(), s_csr.copy()
    pattern.data[:] = 1.0
    s_pat.data[:] = 1.0
    touched = (pattern @ s_pat).toarray() > 0
    cancelled = (touched & (sc == 0)).sum(axis=1)
    assert (sc.view(np.int64)[sc == 0] == 0).all()                          # every zero score is +0
    canc = np.asarray(users["cancel"])
    assert (cancelled[canc] > 0).all()
    assert ((work[canc] <= ie.HASH_WORK) & (sc[canc] != 0).any(axis=1) & (cancelled[canc] > 0)).any()
    assert ((work[canc] > ie.HASH_WORK) & (cancelled[canc] > 0)).any()
    _, dense, _, _ = ie.expected_lists(sc, c["seen"], 100, False)
    ties = 0
    for x, y in c["roles"]["dup"]:
        for u in range(sc.shape[0]):
            row = list(dense[u])
            if x in row and y in row and sc[u, x] != 0:
                assert sc[u, x] == sc[u, y] and row.index(x) < row.index(y)
                ties += 1
    assert ties >= 10
    n = sc.shape[1]
    _, _, _, fsc = ie.expected_lists(sc, c["seen"], n, True)
    for group in ("heavy", "light"):
        mixed = [u for u in users[group] if (fsc[u] > 0).any() and (fsc[u] == 0).any() and (fsc[u] < 0).any()]
        assert len(mixed) >= 3, group


@pytest.mark.parametrize("dense_output", [False, True])
def test_the_similarity_fixture_has_its_structure(dense_output):
    c = ie.sim_case(dense_output)
    rel, mat, users = c["rel"], c["mat"], c["users"]
    off = rel.copy()
    off.setdiag(0)
    off.eliminate_zeros()
    assert (off.data.astype(np.float32).astype(np.float64) != off.data).mean() > 0.99
    assert (off != off.T).nnz > 0.9 * off.nnz                             # not symmetric
    work = ie.score_work(c["p"], mat)
    assert (work[users["heavy"]] > ie.HASH_WORK).all() and (work[users["light"]] <= ie.HASH_WORK).all()
    assert {t: int(work[u]) for t, u in users["work"].items()} == {512: 512, 513: 513}


def test_the_model_case_has_dense_and_sparse_chunks():
    c = ie.model_case()
    assert _bits_equal(c["scores"], io.scores(c["p"], _cooc_matrix(ie.cooc_case()["a"])).toarray())
    modes = io.chunk_modes((c["scores"] != 0).sum(axis=1), ie.COOC_ITEMS, 10, ie.MODEL_LIMIT)
    assert sum(d for _, _, d in modes) >= 3 and sum(not d for _, _, d in modes) >= 3

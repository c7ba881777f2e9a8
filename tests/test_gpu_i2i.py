"""Item-to-item model on the device (pb200_cooc_build, pb200_i2i_topk, B200CooccurrenceModel, dropin_i2i) against the
f64 oracle (oracle/i2i_oracle.py), pb200_topk_dense and the reference's recorded runs (tests/golden/i2i_cases.npz)."""
import os

import numpy as np
import pytest
import scipy.sparse as sps

from oracle import i2i_oracle as io

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "i2i_cases.npz")


@pytest.fixture(scope="module")
def eng():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from polara_b200.engine import get_engine
    return get_engine()


def training(n_users, n_items, seed, signed=False, heavy=True, empty=True, values="int"):
    """random ratings with empty users and items, one item every user rated (a heavy S row) and, with ``signed``,
    +-1 values whose products cancel."""
    rng = np.random.default_rng(seed)
    deg = rng.integers(0, 12, n_users)
    if empty:
        deg[rng.choice(n_users, n_users // 10, replace=False)] = 0
    users = np.repeat(np.arange(n_users), deg)
    pool = n_items - (n_items // 7 if empty else 0)               # the last items are never rated
    items = rng.integers(0, pool, len(users))
    if heavy:
        users = np.r_[users, np.arange(n_users)]
        items = np.r_[items, np.full(n_users, pool // 2)]
    if signed:
        vals = rng.choice([-1.0, 1.0], len(users))
    elif values == "int":
        vals = rng.integers(1, 6, len(users)).astype(np.float64)
    else:
        vals = rng.random(len(users)).astype(np.float32).astype(np.float64) * 4 + 0.25
    a = sps.coo_matrix((vals, (users, items)), shape=(n_users, n_items)).tocsr()
    a.sum_duplicates()
    a.data = a.data.astype(np.float32).astype(np.float64)
    return a


def device_csr(eng, a):
    a = sps.csr_matrix(a)
    a.sort_indices()
    return eng.upload_csr(a.indptr.astype(np.int64), a.indices.astype(np.int32), a.data.astype(np.float32), a.shape)


def oracle_s(a, implicit):
    idx = np.c_[a.tocoo().row, a.tocoo().col]
    return io.cooc_matrix(idx, a.tocoo().data, a.shape, implicit)


@pytest.mark.parametrize("n_users,n_items,implicit,signed", [
    (400, 300, False, False),                  # one panel, n not a multiple of 32
    (400, 300, True, False),
    (700, 2 * 8192 + 77, False, False),        # three column panels, the last one partial
    (700, 2 * 8192 + 77, True, True),
    (900, 8192, False, True),                  # exactly one full panel
])
def test_build_is_exact_on_integer_data(eng, n_users, n_items, implicit, signed):
    from polara_b200.engine import cooc_lds
    a = training(n_users, n_items, 11 + n_items, signed=signed)
    s = eng.cooc_build(device_csr(eng, a), implicit=implicit)
    assert s.shape == (n_items, cooc_lds(n_items))
    got = s[:, :n_items].cpu().numpy()
    want = oracle_s(a, implicit).toarray()
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(got, got.T)
    assert (np.diag(got) == 0).all()
    if signed:
        assert ((a.T @ a).toarray() == 0).sum() > 0          # cancellations happened


def test_build_refuses_a_matrix_larger_than_free_memory(eng):
    import torch
    free = torch.cuda.mem_get_info(eng.device)[0]
    n = int((free / 8) ** 0.5) + 1024
    a = device_csr(eng, sps.csr_matrix(([1.0], ([0], [n - 1])), shape=(2, n)))
    before = torch.cuda.memory_allocated(eng.device)
    with pytest.raises(MemoryError, match="%d items" % n):
        eng.cooc_build(a)
    assert torch.cuda.memory_allocated(eng.device) == before


def make_test_data(n_users, n_items, seed, signed=False, zero_fdbk=True):
    rng = np.random.default_rng(seed)
    deg = rng.integers(0, 9, n_users)
    deg[::13] = 0
    users = np.repeat(np.arange(n_users), deg)
    items = rng.integers(0, n_items, len(users))
    key = np.unique(users * n_items + items)
    users, items = key // n_items, key % n_items
    fd = rng.choice([-1.0, 1.0], len(users)) if signed else rng.integers(1, 6, len(users)).astype(np.float64)
    if zero_fdbk:
        fd[rng.random(len(fd)) < 0.05] = 0.0                    # zero feedback: seen, not in P
    return users, items, fd


def lists_from_oracle(s, users, items, fd, shape, k, filter_seen, implicit):
    p = io.test_matrix(users, items, fd, shape, implicit)
    sc = io.scores(p, s)
    seen = sps.csr_matrix((np.ones(len(users)), (users, items)), shape=shape)
    dense, sparse = np.empty((shape[0], k), np.int64), np.empty((shape[0], k), np.int64)
    full = sc.toarray()
    for u in range(shape[0]):
        sn = seen.indices[seen.indptr[u]:seen.indptr[u + 1]]
        dense[u] = io.dense_rule(full[u], sn, k, filter_seen)
        lo, hi = sc.indptr[u], sc.indptr[u + 1]
        sparse[u] = io.sparse_rule(sc.indices[lo:hi], sc.data[lo:hi], k)
    return np.diff(sc.indptr), dense, sparse, full, seen


def run_topk(eng, s_dev, n_items, users, items, fd, shape, k, filter_seen, implicit, want_scores=False):
    import torch
    from polara_b200.models import _DeviceModelMixin
    mix = _DeviceModelMixin()
    mix._engine = eng
    p_dev, seen_dev = mix._test_csr_device((users, items, fd), shape)
    out = eng.i2i_topk(s_dev, n_items, p_dev, k, seen=seen_dev if filter_seen else None, implicit=implicit,
                       want_scores=want_scores)
    torch.cuda.synchronize()
    return [None if t is None else t.cpu().numpy() for t in out]


@pytest.mark.parametrize("n_items,k,filter_seen,implicit,signed", [
    (300, 10, True, False, False),
    (300, 10, False, False, False),
    (300, 25, True, True, False),
    (1100, 10, True, False, True),             # negative scores and cancellations to exactly 0
    (1100, 10, False, False, True),
    (2 * 8192 + 77, 40, True, False, False),   # many pads, sweep over 65 panels
    (37, 37, True, False, False),              # k = n: the seen items fill the dense list
])
def test_lists_follow_the_oracle_rules_on_integer_data(eng, n_items, k, filter_seen, implicit, signed):
    a = training(500, n_items, 3 + n_items, signed=signed)
    s_dev = eng.cooc_build(device_csr(eng, a), implicit=implicit)
    s = oracle_s(a, implicit)
    shape = (300, n_items)
    users, items, fd = make_test_data(shape[0], n_items, 5 + k, signed=signed)
    nnz, dense, sparse = run_topk(eng, s_dev, n_items, users, items, fd, shape, k, filter_seen, implicit)
    w_nnz, w_dense, w_sparse, full, _ = lists_from_oracle(s, users, items, fd, shape, k, filter_seen, implicit)
    np.testing.assert_array_equal(nnz, w_nnz)
    np.testing.assert_array_equal(dense, w_dense)
    np.testing.assert_array_equal(sparse, w_sparse)
    assert (sparse < 0).any() or n_items == 37
    if signed:
        assert (full < 0).any()


@pytest.mark.parametrize("filter_seen", [True, False])
def test_dense_list_equals_topk_dense_on_the_host_block(eng, filter_seen):
    import torch
    n_items, k = 700, 12
    a = training(600, n_items, 21)
    s_dev = eng.cooc_build(device_csr(eng, a))
    s = oracle_s(a, False)
    shape = (250, n_items)
    users, items, fd = make_test_data(shape[0], n_items, 22)
    _, dense, _, scores = run_topk(eng, s_dev, n_items, users, items, fd, shape, k, filter_seen, False, want_scores=True)
    _, _, _, full, seen = lists_from_oracle(s, users, items, fd, shape, k, filter_seen, False)
    block = eng.upload(np.ascontiguousarray(full))
    sv = (eng.upload(seen.indptr.astype(np.int64)), eng.upload(seen.indices.astype(np.int32))) if filter_seen else None
    ids, sc = eng.topk_dense(block, k, seen=sv, want_scores=True)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(dense, ids.cpu().numpy())
    np.testing.assert_array_equal(scores, sc.cpu().numpy())


def test_non_integer_lists_are_a_valid_topk_of_the_f64_scores(eng):
    """fp32-representable non-integer data: the lists, counts and scores are those of the f64 oracle, bit for bit"""
    n_items, k = 900, 10
    a = training(800, n_items, 31, values="float")
    s_dev = eng.cooc_build(device_csr(eng, a))
    s = oracle_s(a, False)
    shape = (400, n_items)
    users, items, fd = make_test_data(shape[0], n_items, 32, zero_fdbk=False)
    fd = (fd * 0.37).astype(np.float32).astype(np.float64)
    nnz, dense, sparse, scores = run_topk(eng, s_dev, n_items, users, items, fd, shape, k, True, False,
                                          want_scores=True)
    w_nnz, w_dense, w_sparse, full, _ = lists_from_oracle(s, users, items, fd, shape, k, True, False)
    np.testing.assert_array_equal(nnz, w_nnz)
    np.testing.assert_array_equal(dense, w_dense)
    np.testing.assert_array_equal(sparse, w_sparse)
    assert scores.tobytes() == np.take_along_axis(full, w_dense, axis=1).tobytes()


def test_two_runs_give_identical_lists(eng):
    a = training(900, 5000, 41)
    shape = (600, 5000)
    users, items, fd = make_test_data(shape[0], 5000, 42)
    first = None
    for _ in range(2):
        s_dev = eng.cooc_build(device_csr(eng, a))
        got = run_topk(eng, s_dev, 5000, users, items, fd, shape, 20, True, False, want_scores=True)
        if first is None:
            first = got
        else:
            for x, y in zip(first, got):
                assert x.tobytes() == y.tobytes()


def golden_cases():
    return [str(c) for c in np.load(GOLDEN)["cases"]]


@pytest.mark.parametrize("case", golden_cases())
def test_model_reproduces_the_reference_runs(eng, case):
    import pandas as pd
    from polara_b200 import host
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CooccurrenceModel
    g = np.load(GOLDEN)
    p = case + "_"
    hold = pd.DataFrame({"userid": g[p + "holdout_user"], "itemid": g[p + "holdout_item"],
                         "rating": g[p + "holdout_fdbk"]})
    data = ArrayData(g[p + "train_idx"], g[p + "train_val"], g[p + "train_shape"], g[p + "test_user"],
                     g[p + "test_item"], g[p + "test_fdbk"], g[p + "test_shape"], holdout=hold)
    model = B200CooccurrenceModel(data)
    model.verbose = False
    model.topk = int(g[p + "topk"])
    model.filter_seen = bool(g[p + "filter_seen"])
    model.implicit = bool(g[p + "implicit"])
    model.dense_output = bool(g[p + "dense_output"])
    old = host.DEFAULTS["memory_hard_limit"]
    host.DEFAULTS["memory_hard_limit"] = float(g[p + "memory_hard_limit"])
    try:
        model.build()
        recs = model.get_recommendations()
    finally:
        host.DEFAULTS["memory_hard_limit"] = old
    ref = g[p + "recs"]
    a = dict(train_idx=g[p + "train_idx"], train_val=g[p + "train_val"], train_shape=tuple(g[p + "train_shape"]),
             test_user=g[p + "test_user"], test_item=g[p + "test_item"], test_fdbk=g[p + "test_fdbk"],
             test_shape=tuple(g[p + "test_shape"]), topk=model.topk, filter_seen=model.filter_seen,
             implicit=model.implicit, dense_output=model.dense_output,
             memory_hard_limit=float(g[p + "memory_hard_limit"]))
    want, _, _, sc = io.recommend(**a)
    full = sc.toarray()
    rows = np.arange(ref.shape[0])[:, None]
    score = lambda x: np.where(x >= 0, full[rows, np.maximum(x, 0)], np.nan)     # noqa: E731
    np.testing.assert_array_equal(recs < 0, ref < 0)
    seen = sps.csr_matrix((np.ones(len(a["test_user"])), (a["test_user"], a["test_item"])), shape=a["test_shape"])
    flag = lambda x: np.array([np.isin(x[u], seen.indices[seen.indptr[u]:seen.indptr[u + 1]])   # noqa: E731
                               for u in range(x.shape[0])]) & (x >= 0)
    # exact on the float case too: its values are fp32-representable, so S and the scores have the reference's bits
    np.testing.assert_array_equal(score(recs), score(ref))
    np.testing.assert_array_equal(recs, want)                # the oracle's tie rule fixes every id
    np.testing.assert_array_equal(flag(recs), flag(want))


def test_topk_larger_than_the_catalogue_raises(eng):
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CooccurrenceModel
    data = ArrayData(np.array([[0, 0], [0, 1]]), np.array([1.0, 2.0]), (1, 3), np.array([0]), np.array([1]),
                     np.array([1.0]), (1, 3))
    model = B200CooccurrenceModel(data)
    model.verbose = False
    model.build()
    model.topk = 4
    with pytest.raises(ValueError):
        model.get_recommendations()


def test_dropin_matches_polaras_own_cooccurrence_model():
    pd = pytest.importorskip("pandas")
    from oracle import ref_driver as rd
    if rd.reference_root() is None:
        pytest.skip("reference not installed (oracle/_ref)")
    rd.import_reference()
    from polara.recommender.data import RecommenderData
    from polara.recommender.models import CooccurrenceModel
    from polara_b200.models import dropin_i2i
    from polara_b200.synth import planted_ratings
    u, i, r = planted_ratings(1200, 900, 12, rank=6, seed=23)
    data = RecommenderData(pd.DataFrame({"userid": u, "itemid": i, "rating": r.astype(np.int64)}), "userid", "itemid",
                           "rating", seed=0)
    data.verbose = False
    data.prepare()
    ref = CooccurrenceModel(data)
    ref.verbose = False
    ref.build()
    ref_recs = ref.get_recommendations()
    mine = dropin_i2i()(data)
    mine.verbose = False
    mine.build()
    recs = mine.get_recommendations()
    assert recs.shape == ref_recs.shape and recs.dtype == ref_recs.dtype
    np.testing.assert_array_equal(recs < 0, ref_recs < 0)
    test_data, shape, _ = ref._get_test_data()
    s = ref._i2i_matrix
    p = ref.get_test_matrix(test_data, shape)[0].astype(np.float64)
    full = np.asarray((p @ s).todense())
    rows = np.arange(shape[0])[:, None]
    np.testing.assert_array_equal(np.where(recs >= 0, full[rows, np.maximum(recs, 0)], 0),
                                  np.where(ref_recs >= 0, full[rows, np.maximum(ref_recs, 0)], 0))
    # the same scores position by position; ties at the cut may still swap items
    assert abs(ref.evaluate("hits").true_positive - mine.evaluate("hits").true_positive) <= 3

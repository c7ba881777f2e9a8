"""Sparse storage of the item-to-item matrix (pb200_cooc_build_csr, pb200_i2i_topk_csr, the ``storage`` of the
item-to-item models) against the dense path (pb200_cooc_build, pb200_i2i_topk), scipy, the f64 oracles and the
reference's recorded runs; and B200SimilarityAggregation / dropin_similarity against tests/golden/sim_cases.npz."""
import os

import numpy as np
import pytest
import scipy.sparse as sps

from oracle import i2i_oracle as io
from oracle import sim_oracle as so
from tests.test_gpu_i2i import device_csr, make_test_data, oracle_s, run_topk, training

pytestmark = pytest.mark.gpu

SIM = os.path.join(os.path.dirname(__file__), "golden", "sim_cases.npz")
WIDE = os.path.join(os.path.dirname(__file__), "golden", "i2i_wide_cases.npz")
HASH_WORK = 512            # rows / users with more work than this take the global-row path (csrc/i2i.cu kHashWork)


@pytest.fixture(scope="module")
def eng():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from polara_b200.engine import get_engine
    return get_engine()


@pytest.fixture
def free_probe(eng, monkeypatch):
    """records every free-memory reading the builds take (the real probe underneath)"""
    seen = []
    real = eng.free_bytes

    def probe():
        v = real()
        seen.append(v)
        return v
    monkeypatch.setattr(eng, "free_bytes", probe)
    return seen


def host_csr(s):
    import torch
    torch.cuda.synchronize()
    return sps.csr_matrix((s.values.cpu().numpy(), s.indices.cpu().numpy(), s.indptr.cpu().numpy()), shape=s.shape)


def build_work(a):
    """work of each item row: sum over its users of their row lengths"""
    lens = np.diff(a.indptr)
    at = a.T.tocsr()
    return np.array([lens[at.indices[at.indptr[i]:at.indptr[i + 1]]].sum() for i in range(a.shape[1])])


def check_pattern(c, n):
    for i in range(n):
        cols = c.indices[c.indptr[i]:c.indptr[i + 1]]
        assert (np.diff(cols) > 0).all() and i not in cols
    assert (c.data != 0).all()


@pytest.mark.parametrize("n_users,n_items,implicit,signed", [
    (400, 300, False, False),
    (400, 300, True, False),
    (700, 2 * 8192 + 77, False, False),        # three dense column panels, the last one partial
    (700, 2 * 8192 + 77, True, True),
    (900, 8192, False, True),                  # one full panel; +-1 products cancel
])
def test_csr_build_equals_the_dense_build_bit_for_bit(eng, n_users, n_items, implicit, signed):
    a = training(n_users, n_items, 11 + n_items, signed=signed)
    work = build_work(a)
    assert work.max() > HASH_WORK and ((work > 0) & (work <= HASH_WORK)).any()       # both accumulator paths
    d = device_csr(eng, a)
    c = host_csr(eng.cooc_build_csr(d, implicit=implicit))
    dense = eng.cooc_build(d, implicit=implicit)[:, :n_items].cpu().numpy()
    rows = np.repeat(np.arange(n_items), np.diff(c.indptr))
    assert c.data.tobytes() == dense[rows, c.indices].tobytes()
    outside = dense.copy()
    outside[rows, c.indices] = 0
    assert not outside.any()
    check_pattern(c, n_items)
    if signed:
        want = oracle_s(a, implicit)
        assert want.nnz == c.nnz and ((a.T @ a).toarray() == 0).sum() > 0


def test_csr_build_of_a_hub_item_matches_scipy(eng):
    rng = np.random.default_rng(5)
    m, n = 3000, 4000
    users = np.repeat(np.arange(m), rng.integers(1, 8, m))
    items = rng.integers(1, n, len(users))
    users, items = np.r_[users, np.arange(m)], np.r_[items, np.zeros(m, np.int64)]    # item 0: every user
    a = sps.coo_matrix((rng.integers(1, 6, len(users)).astype(np.float64), (users, items)), shape=(m, n)).tocsr()
    a.sum_duplicates()
    assert build_work(a)[0] > 10 * HASH_WORK
    c = host_csr(eng.cooc_build_csr(device_csr(eng, a)))
    want = (a.T @ a).tocsr()
    want.setdiag(0)
    want.eliminate_zeros()
    want.sort_indices()
    assert c.indptr.tolist() == want.indptr.tolist() and c.indices.tolist() == want.indices.tolist()
    assert c.data.tobytes() == want.data.tobytes()
    assert np.diff(c.indptr)[0] > 1000


def scoring_data(n_users, n_items, seed, signed):
    """make_test_data plus four users of 120 items each: their work takes the global-row scoring path"""
    users, items, fd = make_test_data(n_users, n_items, seed, signed=signed)
    rng = np.random.default_rng(seed + 1)
    hu = np.repeat(np.arange(0, n_users, n_users // 4), 120)
    hi = rng.integers(0, n_items, len(hu))
    hf = rng.choice([-1.0, 1.0], len(hu)) if signed else rng.integers(1, 6, len(hu)).astype(np.float64)
    key, first = np.unique(np.r_[users * n_items + items, hu * n_items + hi], return_index=True)
    return key // n_items, key % n_items, np.r_[fd, hf][first]


@pytest.mark.parametrize("k", [1, 10, 100])
@pytest.mark.parametrize("filter_seen,implicit,signed", [
    (True, False, False), (False, False, False), (True, True, False), (True, False, True), (False, False, True)])
def test_csr_scoring_equals_the_dense_scoring(eng, k, filter_seen, implicit, signed):
    n_items = 1100
    a = training(500, n_items, 3 + k, signed=signed)
    d = device_csr(eng, a)
    s_dense = eng.cooc_build(d, implicit=implicit)
    s_csr = eng.cooc_build_csr(d, implicit=implicit)
    shape = (300, n_items)
    users, items, fd = scoring_data(shape[0], n_items, 5 + k, signed)
    want = run_topk(eng, s_dense, n_items, users, items, fd, shape, k, filter_seen, implicit, want_scores=True)
    from polara_b200.models import _DeviceModelMixin
    mix = _DeviceModelMixin()
    mix._engine = eng
    p_dev, seen_dev = mix._test_csr_device((users, items, fd), shape)
    got = eng.i2i_topk_csr(s_csr, p_dev, k, seen=seen_dev if filter_seen else None, implicit=implicit,
                           want_scores=True)
    got = [t.cpu().numpy() for t in got]
    for x, y in zip(got, want):
        assert x.tobytes() == y.tobytes()
    assert (got[0] < k).any()                                   # users with fewer than k nonzero scores
    p = io.test_matrix(users, items, fd, shape, implicit)
    s_host = host_csr(s_csr)
    work = np.array([np.diff(s_host.indptr)[p.indices[p.indptr[u]:p.indptr[u + 1]]].sum() for u in range(shape[0])])
    assert work.max() > HASH_WORK and (work <= HASH_WORK).any()


def test_two_builds_and_scorings_give_identical_bits(eng):
    a = training(900, 5000, 41, signed=True)
    shape = (600, 5000)
    users, items, fd = scoring_data(shape[0], 5000, 42, True)
    from polara_b200.models import _DeviceModelMixin
    mix = _DeviceModelMixin()
    mix._engine = eng
    runs = []
    for _ in range(2):
        s = eng.cooc_build_csr(device_csr(eng, a))
        p_dev, seen_dev = mix._test_csr_device((users, items, fd), shape)
        out = eng.i2i_topk_csr(s, p_dev, 20, seen=seen_dev, want_scores=True)
        runs.append([t.cpu().numpy().tobytes() for t in (s.indptr, s.indices, s.values) + tuple(out)])
    assert runs[0] == runs[1]


def wide_training(n_users, n_items, per_user, seed):
    rng = np.random.default_rng(seed)
    users = np.repeat(np.arange(n_users), per_user)
    items = rng.integers(0, n_items, len(users))
    key = np.unique(users * n_items + items)
    return np.c_[key // n_items, key % n_items], rng.integers(1, 6, len(key)).astype(np.float64)


def test_auto_storage_goes_sparse_beyond_dense_reach(eng, free_probe):
    from polara_b200.engine import cooc_lds
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CooccurrenceModel
    n_users, n_items = 20000, 150_000
    idx, val = wide_training(n_users, n_items, 6, 3)
    tu, ti, tf = make_test_data(2000, n_items, 4, zero_fdbk=False)
    data = ArrayData(idx, val, (n_users, n_items), tu, ti, tf, (2000, n_items))
    model = B200CooccurrenceModel(data)
    model.verbose = False
    model.build()
    assert model.storage == "auto" and model.i2i_storage == "sparse"
    assert free_probe and n_items * cooc_lds(n_items) * 8 > max(free_probe)       # dense S: 180 GB
    nnz, dense, sparse = model.i2i_lists((tu, ti, tf), (2000, n_items))
    s = io.cooc_matrix(idx, val, (n_users, n_items))
    p = io.test_matrix(tu, ti, tf, (2000, n_items))
    sc = io.scores(p, s)
    seen = sps.csr_matrix((np.ones(len(tu)), (tu, ti)), shape=(2000, n_items))
    np.testing.assert_array_equal(nnz, np.diff(sc.indptr))
    for u in np.random.default_rng(0).choice(2000, 60, replace=False):
        lo, hi = sc.indptr[u], sc.indptr[u + 1]
        row = np.zeros(n_items)
        row[sc.indices[lo:hi]] = sc.data[lo:hi]
        np.testing.assert_array_equal(dense[u], io.dense_rule(row, seen.indices[seen.indptr[u]:seen.indptr[u + 1]], 10))
        np.testing.assert_array_equal(sparse[u], io.sparse_rule(sc.indices[lo:hi], sc.data[lo:hi], 10))
    recs = model.get_recommendations()
    assert recs.shape == (2000, 10)


def test_dense_storage_keeps_the_refusal(eng):
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CooccurrenceModel
    idx, val = wide_training(200, 150_000, 3, 5)
    model = B200CooccurrenceModel(ArrayData(idx, val, (200, 150_000)))
    model.verbose = False
    model.storage = "dense"
    with pytest.raises(MemoryError, match="dense item x item matrix of 150000 items"):
        model.build()


def test_csr_refusal_leaves_nothing_allocated(eng, monkeypatch):
    import torch
    from polara_b200 import engine as engine_mod
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CooccurrenceModel
    real = engine_mod.cooc_csr_memory_check
    counted = []

    def tiny_after_count(nnz, n_items, scratch, free):
        if nnz:                                       # the counted CSR meets a tiny free-byte count
            counted.append(nnz)
            free = 4096
        return real(nnz, n_items, scratch, free)
    monkeypatch.setattr(engine_mod, "cooc_csr_memory_check", tiny_after_count)
    a = training(400, 3000, 7)
    d = device_csr(eng, a)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(eng.device)
    with pytest.raises(MemoryError, match="sparse item x item matrix of 3000 items with"):
        eng.cooc_build_csr(d)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(eng.device) == before and counted == [oracle_s(a, False).nnz]
    idx = np.c_[a.tocoo().row, a.tocoo().col]
    model = B200CooccurrenceModel(ArrayData(idx, a.tocoo().data, a.shape))
    model.verbose = False
    model.storage = "sparse"
    with pytest.raises(MemoryError):
        model.build()


def test_sparse_storage_reproduces_the_wide_reference_run(eng):
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CooccurrenceModel
    w = np.load(WIDE)
    p = "wide_"
    data = ArrayData(w[p + "train_idx"], w[p + "train_val"], w[p + "train_shape"], w[p + "test_user"],
                     w[p + "test_item"], w[p + "test_fdbk"], w[p + "test_shape"])
    recs = {}
    for storage in ("sparse", "dense"):
        model = B200CooccurrenceModel(data)
        model.verbose = False
        model.storage = storage
        model.build()
        assert model.i2i_storage == storage
        recs[storage] = model.get_recommendations()
    np.testing.assert_array_equal(recs["sparse"], recs["dense"])
    want = io.recommend(w[p + "train_idx"], w[p + "train_val"], tuple(w[p + "train_shape"]), w[p + "test_user"],
                        w[p + "test_item"], w[p + "test_fdbk"], tuple(w[p + "test_shape"]))[0]
    np.testing.assert_array_equal(recs["sparse"], want)
    np.testing.assert_array_equal(recs["sparse"] < 0, w[p + "recs"] < 0)


def sim_cases():
    return [str(c) for c in np.load(SIM)["cases"]]


@pytest.mark.parametrize("case", sim_cases())
def test_similarity_model_reproduces_the_reference_runs(eng, case):
    import pandas as pd
    from polara_b200 import host
    from polara_b200.host import ArrayData
    from polara_b200.models import B200SimilarityAggregation
    g = np.load(SIM)
    p = case + "_"
    rel = sps.csr_matrix((g[p + "rel_data"], g[p + "rel_indices"], g[p + "rel_indptr"]),
                         shape=tuple(g[p + "rel_shape"]))
    shape = tuple(g[p + "test_shape"])
    hold = pd.DataFrame({"userid": g[p + "holdout_user"], "itemid": g[p + "holdout_item"],
                         "rating": g[p + "holdout_fdbk"]})
    data = ArrayData(np.zeros((0, 2), np.int64), np.zeros(0), shape, g[p + "test_user"], g[p + "test_item"],
                     g[p + "test_fdbk"], shape, holdout=hold, item_relations=rel)
    model = B200SimilarityAggregation(data)
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
    assert (rel.diagonal() == 1).all() and (data.item_relations.diagonal() == 1).all()     # the copy was edited
    ref = g[p + "recs"]
    want, _, _, sc = so.recommend(rel, g[p + "test_user"], g[p + "test_item"], g[p + "test_fdbk"], shape,
                                  topk=model.topk, filter_seen=model.filter_seen, implicit=model.implicit,
                                  dense_output=model.dense_output, memory_hard_limit=float(g[p + "memory_hard_limit"]))
    full = sc.toarray()
    rows = np.arange(ref.shape[0])[:, None]
    score = lambda x: np.where(x >= 0, full[rows, np.maximum(x, 0)], np.nan)     # noqa: E731
    np.testing.assert_array_equal(recs < 0, ref < 0)
    # exact on the float case too: the device reads the fp64 relations unrounded and sums them in scipy's order
    np.testing.assert_array_equal(score(recs), score(ref))
    np.testing.assert_array_equal(recs, want)


def test_dropin_similarity_matches_polaras_own_model():
    pd = pytest.importorskip("pandas")
    from oracle import ref_driver as rd
    if rd.reference_root() is None:
        pytest.skip("reference not installed (oracle/_ref)")
    rd.import_reference()
    from polara.recommender.hybrid.data import SimilarityDataModel
    from polara.recommender.hybrid.models import SimilarityAggregation
    from polara_b200.models import dropin_similarity
    from polara_b200.synth import planted_ratings
    u, i, r = planted_ratings(1200, 900, 12, rank=6, seed=23)
    rng = np.random.default_rng(1)
    nz = 8000
    rel = sps.coo_matrix((rng.integers(1, 6, nz).astype(np.float64), (rng.integers(0, 900, nz),
                          rng.integers(0, 900, nz))), shape=(900, 900)).tocsr()
    data = SimilarityDataModel(pd.DataFrame({"userid": u, "itemid": i, "rating": r.astype(np.int64)}), "userid",
                               "itemid", "rating", seed=0, relations_matrices={"itemid": rel},
                               relations_indices={"itemid": np.arange(900)})
    data.verbose = False
    data.prepare()
    ref = SimilarityAggregation(data)
    ref.verbose = False
    ref.build()
    ref_recs = ref.get_recommendations()
    mine = dropin_similarity()(data)
    mine.verbose = False
    mine.build()
    recs = mine.get_recommendations()
    assert recs.shape == ref_recs.shape and recs.dtype == ref_recs.dtype
    test_data, shape, _ = ref._get_test_data()
    p = ref.get_test_matrix(test_data, shape)[0].astype(np.float64)
    full = np.asarray((p @ ref.item_similarity_matrix.T).todense())
    rows = np.arange(shape[0])[:, None]
    np.testing.assert_array_equal(recs < 0, ref_recs < 0)
    np.testing.assert_array_equal(np.where(recs >= 0, full[rows, np.maximum(recs, 0)], 0),
                                  np.where(ref_recs >= 0, full[rows, np.maximum(ref_recs, 0)], 0))


def test_nothing_co_occurs(eng):
    """every user rated one item: S has no entry; the CSR is empty and scores like the all-zero dense S"""
    import torch
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CooccurrenceModel
    n_users, n_items = 500, 700
    rng = np.random.default_rng(9)
    a = sps.csr_matrix((rng.integers(1, 6, n_users).astype(np.float64), (np.arange(n_users),
                        rng.integers(0, n_items, n_users))), shape=(n_users, n_items))
    d = device_csr(eng, a)
    s_csr = eng.cooc_build_csr(d)
    s_dense = eng.cooc_build(d)
    torch.cuda.synchronize()
    assert s_csr.nnz == 0 and not s_csr.indptr.cpu().numpy().any() and s_csr.values.dtype == torch.float64
    assert not s_dense[:, :n_items].cpu().numpy().any()
    users, items, fd = make_test_data(200, n_items, 10)
    want = run_topk(eng, s_dense, n_items, users, items, fd, (200, n_items), 10, True, False, want_scores=True)
    from polara_b200.models import _DeviceModelMixin
    mix = _DeviceModelMixin()
    mix._engine = eng
    p_dev, seen_dev = mix._test_csr_device((users, items, fd), (200, n_items))
    got = [t.cpu().numpy() for t in eng.i2i_topk_csr(s_csr, p_dev, 10, seen=seen_dev, want_scores=True)]
    for x, y in zip(got, want):
        assert x.tobytes() == y.tobytes()
    assert not got[0].any() and (got[2] == -1).all()
    idx = np.c_[a.tocoo().row, a.tocoo().col]
    recs = {}
    for storage in ("sparse", "dense"):
        model = B200CooccurrenceModel(ArrayData(idx, a.tocoo().data, a.shape, users, items, fd, (200, n_items)))
        model.verbose = False
        model.storage = storage
        model.build()
        recs[storage] = model.get_recommendations()
    np.testing.assert_array_equal(recs["sparse"], recs["dense"])


def test_scoring_refuses_when_its_scratch_does_not_fit(eng, monkeypatch):
    import torch
    a = training(300, 400, 13)
    s_csr = eng.cooc_build_csr(device_csr(eng, a))
    from polara_b200.models import _DeviceModelMixin
    mix = _DeviceModelMixin()
    mix._engine = eng
    users, items, fd = make_test_data(100, 400, 14)
    p_dev, seen_dev = mix._test_csr_device((users, items, fd), (100, 400))
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(eng.device)
    monkeypatch.setattr(eng, "free_bytes", lambda: 4096)
    with pytest.raises(MemoryError, match="100 test users at k = 10"):
        eng.i2i_topk_csr(s_csr, p_dev, 10, seen=seen_dev)
    assert torch.cuda.memory_allocated(eng.device) == before


def test_fp64_csr_is_refused_where_fp32_values_are_read(eng):
    a = training(300, 400, 15)
    s_csr = eng.cooc_build_csr(device_csr(eng, a))
    with pytest.raises(TypeError):
        s_csr.view()
    with pytest.raises(TypeError):
        eng.transpose(s_csr)

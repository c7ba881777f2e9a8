"""The item-to-item kernels (pb200_cooc_build, pb200_cooc_build_csr, pb200_i2i_topk, pb200_i2i_topk_csr) bit for bit
against the exact host emulation of their summation order (tests/i2i_exact.py), on non-integer data whose sums depend
on that order, on both accumulator paths of the sparse kernels and with their global rows reused.  Every case runs
twice and the second run must give the same bits."""
import numpy as np
import pytest

from oracle import i2i_oracle as io
from tests import i2i_exact as ie
from tests.test_gpu_i2i import device_csr, run_topk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from polara_b200.engine import get_engine
    return get_engine()


def host(*tensors):
    import torch
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in tensors]


def twice(run):
    """run() twice; the outputs (lists of arrays) must have the same bits"""
    first, second = run(), run()
    for x, y in zip(first, second):
        assert x.tobytes() == y.tobytes()
    return first


def assert_bits(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, got.dtype, want.shape, want.dtype)
    if got.tobytes() != want.tobytes():
        bad = np.asarray(got != want) if got.dtype.kind != "f" else ie.differs(got, want)
        pytest.fail("%s: %d of %d entries differ, first at %s" % (what, bad.sum(), bad.size, np.argwhere(bad)[0]))


# ---- build -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("panel_cols", [100, 1000, 8192])
def test_dense_build_is_the_emulated_sum(eng, monkeypatch, panel_cols):
    """S[:, :n] of 15, 2 and 1 column panels (the last one partial) against build_s; symmetric, +0 diagonal and +0
    where the products cancel"""
    c = ie.cooc_case()
    n = ie.COOC_ITEMS
    monkeypatch.setattr(eng, "COOC_PANEL_COLS", panel_cols)
    d = device_csr(eng, c["a"])
    s, = twice(lambda: host(eng.cooc_build(d)[:, :n]))
    assert_bits(s, c["s"], "S")
    assert s.tobytes() == np.ascontiguousarray(s.T).tobytes()
    assert (np.diag(s).view(np.int64) == 0).all()
    for i, j in c["roles"]["cancel"]:
        assert s[i, j].view(np.int64) == 0 and s[j, i].view(np.int64) == 0


def test_dense_build_at_the_full_panel_width(eng):
    """8525 items: two panels of 8192 columns, the last one partial; the emulated rows"""
    import torch
    w = ie.wide_case()
    n, rows = ie.WIDE_ITEMS, w["rows"]
    assert eng.COOC_PANEL_COLS == 8192 and n % 8192
    d = device_csr(eng, w["a"])
    sel = torch.as_tensor(rows, device=eng.device)

    def run():
        s = eng.cooc_build(d)
        return host(s.index_select(0, sel)[:, :n])
    s, = twice(run)
    assert_bits(s, w["s"], "S rows")
    assert s[:, rows].tobytes() == np.ascontiguousarray(s[:, rows].T).tobytes()
    assert (s[np.arange(len(rows)), rows].view(np.int64) == 0).all()


@pytest.mark.parametrize("acc_rows", [None, 1, 3])
def test_csr_build_is_the_emulated_sum(eng, monkeypatch, acc_rows):
    """indptr, indices and values of pb200_cooc_build_csr against the CSR of build_s.  With 1 or 3 global rows a CTA
    accumulates many long rows in turn, each on the row its predecessor cleared behind the read."""
    c = ie.cooc_case()
    if acc_rows is not None:
        monkeypatch.setattr(eng, "COOC_CSR_ACC_ROWS", acc_rows)
    work = ie.build_work(c["a"])
    sensitive = ie.differs(c["s"], ie.build_s(c["a"], order="desc")).any(axis=1)
    assert (sensitive & (work > 0) & (work <= ie.HASH_WORK)).sum() >= 100
    assert (sensitive & (work > ie.HASH_WORK)).sum() >= 10 * (acc_rows or 1)
    d = device_csr(eng, c["a"])

    def run():
        s = eng.cooc_build_csr(d)
        return host(s.indptr, s.indices, s.values)
    indptr, indices, values = twice(run)
    want = c["s_csr"]
    assert_bits(indptr, want.indptr.astype(np.int64), "indptr")
    assert_bits(indices, want.indices.astype(np.int32), "indices")
    assert_bits(values, want.data, "values")


# ---- scoring ---------------------------------------------------------------------------------------------------------
def csr_topk(eng, s_csr, triplets, shape, k, filter_seen):
    from polara_b200.models import _DeviceModelMixin
    mix = _DeviceModelMixin()
    mix._engine = eng
    p_dev, seen_dev = mix._test_csr_device(triplets, shape)
    return host(*eng.i2i_topk_csr(s_csr, p_dev, k, seen=seen_dev if filter_seen else None, want_scores=True))


def assert_lists(got, want, what):
    for x, y, name in zip(got, want, ("nnz", "dense", "sparse", "scores")):
        assert_bits(x, y, "%s %s" % (what, name))


@pytest.mark.parametrize("k", [1, 10, 100, ie.COOC_ITEMS])
@pytest.mark.parametrize("filter_seen", [True, False])
def test_scoring_is_the_emulated_sum(eng, k, filter_seen):
    """pb200_i2i_topk and pb200_i2i_topk_csr: nnz_u, both rules' lists and the dense lists' scores against the emulated
    scores under the oracle's rules, on the table and the global-row path; six sweep panels, the last one partial"""
    c = ie.cooc_case()
    n = ie.COOC_ITEMS
    d = device_csr(eng, c["a"])
    s_dense = eng.cooc_build(d)
    s_csr = eng.cooc_build_csr(d)
    want = ie.expected_lists(c["scores"], c["seen"], k, filter_seen)
    dense = twice(lambda: run_topk(eng, s_dense, n, *c["triplets"], c["shape"], k, filter_seen, False,
                                   want_scores=True))
    assert_lists(dense, want, "i2i_topk")
    sparse = twice(lambda: csr_topk(eng, s_csr, c["triplets"], c["shape"], k, filter_seen))
    assert_lists(sparse, want, "i2i_topk_csr")
    work = ie.score_work(c["p"], c["s_csr"])
    assert (work <= ie.HASH_WORK).sum() >= 100 and (work > ie.HASH_WORK).sum() >= 40


@pytest.mark.parametrize("k", [10, ie.COOC_ITEMS])
@pytest.mark.parametrize("filter_seen", [True, False])
def test_csr_scoring_with_one_global_row(eng, monkeypatch, k, filter_seen):
    """one warp scores every long user in turn, each on the row the previous user's clearing left zero"""
    c = ie.cooc_case()
    monkeypatch.setattr(eng, "I2I_CSR_ACC_ROWS", 1)
    s_csr = eng.cooc_build_csr(device_csr(eng, c["a"]))
    got = twice(lambda: csr_topk(eng, s_csr, c["triplets"], c["shape"], k, filter_seen))
    assert_lists(got, ie.expected_lists(c["scores"], c["seen"], k, filter_seen), "i2i_topk_csr, one row")


@pytest.mark.parametrize("k", [10, 100])
@pytest.mark.parametrize("dense_output", [False, True])
def test_similarity_operand_scoring_is_the_emulated_sum(eng, dense_output, k):
    """SimilarityAggregation's operand (Sᵀ, or S with ``dense_output``) of non-symmetric relations with arbitrary fp64
    values, read unrounded, through pb200_i2i_topk_csr"""
    from polara_b200.engine import DeviceCSR
    c = ie.sim_case(dense_output)
    mat = c["mat"]
    m_dev = DeviceCSR(eng.upload(mat.indptr.astype(np.int64)), eng.upload(mat.indices.astype(np.int32)),
                      eng.upload(mat.data), mat.shape)
    got = twice(lambda: csr_topk(eng, m_dev, c["triplets"], c["shape"], k, True))
    assert_lists(got, ie.expected_lists(c["scores"], c["seen"], k, True), "similarity operand")


def test_model_storages_reproduce_the_oracle_on_non_integer_data(eng):
    """B200CooccurrenceModel, dense and sparse storage, with chunks of both rules: get_recommendations() equals
    io.recommend"""
    from polara_b200 import host as host_mod
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CooccurrenceModel
    a, c = ie.cooc_case()["a"], ie.model_case()
    coo = a.tocoo()
    idx = np.c_[coo.row, coo.col]
    user, item, fdbk = c["triplets"]
    want, modes, _, _ = io.recommend(idx, coo.data, a.shape, user, item, fdbk, c["shape"], topk=10,
                                     memory_hard_limit=ie.MODEL_LIMIT)
    assert {d for _, _, d in modes} == {True, False}
    recs = {}
    old = host_mod.DEFAULTS["memory_hard_limit"]
    host_mod.DEFAULTS["memory_hard_limit"] = ie.MODEL_LIMIT
    try:
        for storage in ("dense", "sparse"):
            model = B200CooccurrenceModel(ArrayData(idx, coo.data, a.shape, user, item, fdbk, c["shape"]))
            model.verbose = False
            model.storage = storage
            model.build()
            assert model.i2i_storage == storage
            recs[storage], = twice(lambda: [model.get_recommendations()])
    finally:
        host_mod.DEFAULTS["memory_hard_limit"] = old
    assert_bits(recs["dense"], want, "dense storage")
    assert_bits(recs["sparse"], recs["dense"], "sparse storage")

"""The host emulation of the scaled training matrix and of the dense downvote (tests/scaled_exact.py) against the
reference's own outputs, bit for bit: the runs recorded by oracle/make_scaling_golden.py into
tests/golden/scaling_cases.npz and, where the reference is installed under oracle/_ref, the reference run live on fresh
cases.  Also the oracle's and the host path's scaling against the same records.  CPU only."""
import numpy as np
import pytest
import scipy.sparse as sps

from oracle import polara_oracle as po
from oracle.ref_driver import StubData, import_reference, reference_root
from tests import scaled_exact as se


@pytest.fixture(scope="module")
def g(golden):
    return golden("scaling_cases")


def _cases():
    import os
    path = os.path.join(os.path.dirname(__file__), "golden", "scaling_cases.npz")
    return [str(c) for c in np.load(path)["cases"]]


def _bits(x):
    return np.asarray(x, np.float64).view(np.int64)


def _recorded(g, key):
    n = len(g[key + "_indptr"]) - 1
    return g[key + "_indptr"], g[key + "_indices"], g[key + "_data"], n


def _case(g, c):
    p = c + "_"
    return (g[p + "idx"], g[p + "val"], tuple(g[p + "shape"]), float(g[p + "row_scaling"]),
            float(g[p + "col_scaling"]))


def check_against(base_ref, rows_ref, scaled_ref, idx, val, shape, rs, cs):
    """the emulation against the reference's unscaled matrix, row pass and scaled matrix (scipy CSRs, sorted)."""
    base = se.reference_csr(idx, val, shape)
    np.testing.assert_array_equal(base.indptr, base_ref.indptr)
    np.testing.assert_array_equal(base.indices, base_ref.indices)
    assert np.array_equal(_bits(base.data), _bits(base_ref.data)), "unscaled values (signed zeros included)"
    out, kept, rf, _ = se.reference_scaled(base, rs, cs)
    rows = np.repeat(np.arange(shape[0]), np.diff(base.indptr))
    for ref in (rows_ref, scaled_ref):
        # the reference's passes store only nonzero results: its pattern is the kept part of the unscaled one
        np.testing.assert_array_equal(ref.indptr, np.r_[0, np.cumsum(np.bincount(rows[kept], minlength=shape[0]))])
        np.testing.assert_array_equal(ref.indices, base.indices[kept])
    assert np.array_equal(_bits((base.data * rf[rows])[kept]), _bits(rows_ref.data)), "row pass"
    assert np.array_equal(_bits(out[kept]), _bits(scaled_ref.data)), "scaled values"
    assert not out[~kept].any()


@pytest.mark.parametrize("case", _cases())
def test_emulation_matches_recorded_reference(g, case):
    idx, val, shape, rs, cs = _case(g, case)
    mats = {}
    for key in ("base", "rows", "scaled"):
        indptr, indices, data, n = _recorded(g, case + "_" + key)
        mats[key] = sps.csr_matrix((data, indices, indptr), shape=shape)
    check_against(mats["base"], mats["rows"], mats["scaled"], idx, val, shape, rs, cs)
    if case != "example":
        # what the case is there for: stored zeros, and columns whose count changes once they are dropped
        base = mats["base"]
        assert (base.data == 0).sum() > 50 and np.diff(base.indptr).max() > 32
        assert (np.bincount(base.indices, minlength=shape[1]) != np.bincount(mats["scaled"].indices, minlength=shape[1])).sum() > 5


@pytest.mark.parametrize("case", _cases())
def test_oracle_and_host_scaling_match_recorded_reference(g, case):
    """po.scaled_training_matrix and the host path of ScaledHybridSVD (models._rescale_host) on the reference's unscaled
    matrix give the reference's scaled matrix, bit for bit and without stored zeros."""
    from polara_b200.models import _rescale_host
    _, _, shape, rs, cs = _case(g, case)
    indptr, indices, data, _ = _recorded(g, case + "_base")
    base = sps.csr_matrix((data.astype(np.float64), indices, indptr), shape=shape)
    s_ptr, s_idx, s_data, _ = _recorded(g, case + "_scaled")
    for got in (po.scaled_training_matrix(base, rs, cs), _rescale_host(_rescale_host(base.copy(), rs, 1), cs, 0)):
        got.sort_indices()
        np.testing.assert_array_equal(got.indptr, s_ptr)
        np.testing.assert_array_equal(got.indices, s_idx)
        assert np.array_equal(_bits(got.data), _bits(s_data))


def test_example_from_the_column_counts(g):
    """feedback (0,0)=1, (0,1)=0, (1,1)=2, (1,2)=3, (2,1)=0, (2,0)=1, (2,0)=-1, (3,1)=5 at (1, 0.4): column 1 has one
    nonzero (and two stored zeros), so its factor is 1 and not 3 ** -0.3."""
    indptr, indices, data, _ = _recorded(g, "example_scaled")
    dense = sps.csr_matrix((data, indices, indptr), shape=(4, 3)).toarray()
    np.testing.assert_allclose(dense[1], [0, 2 * 2 ** -0.3, 3], rtol=1e-15)
    assert dense[0, 0] == 1.0


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_downvote_emulation_matches_recorded_reference(g, dtype):
    p = "dv_%s_" % dtype
    s = g[p + "scores"]
    assert s.dtype == np.dtype(dtype)
    got = se.reference_downvote(s, g[p + "rows"], g[p + "cols"])
    assert got.dtype == s.dtype
    assert np.array_equal(got.view(np.uint8), g[p + "lowered"].view(np.uint8))


def test_reference_csr_refuses_order_dependent_runs():
    idx = np.zeros((3, 2), np.int64)
    with pytest.raises(AssertionError):
        se.reference_csr(idx, np.array([1.0, 1e-17, -1.0]), (1, 1))
    with pytest.raises(AssertionError):
        se.reference_csr(idx, np.array([1.0, 2 ** -30, 3.0], np.float32), (1, 1))
    # a dyadic triple and a pair are fine; drop_zeros filters before summing, so +x, -x leaves a stored zero
    a = se.reference_csr(np.zeros((5, 2), np.int64), np.array([0.25, 0.0, -1.5, 0.375, 0.0]), (1, 1), drop_zeros=True)
    assert a.nnz == 1 and a.data[0] == -0.875
    b = se.reference_csr(np.zeros((2, 2), np.int64), np.array([0.1, -0.1]), (1, 1), drop_zeros=True)
    assert b.nnz == 1 and b.data[0] == 0


# ---------------------------------------------------------------------------------------------------------------------
#  live: the reference installed under oracle/_ref, on cases the records do not hold
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def reference():
    if reference_root() is None:
        pytest.skip("the reference is not installed under oracle/_ref")
    import_reference()
    from polara.preprocessing.matrices import rescale_matrix
    from polara.recommender.models import RecommenderModel, ScaledSVD, SVDModel
    return rescale_matrix, RecommenderModel, ScaledSVD, SVDModel


@pytest.mark.parametrize("rs,cs", [(1, 0.4), (0.8, 0.4), (1.3, 0), (0.5, 1)])
@pytest.mark.parametrize("dtype,sorted_input", [(np.float32, False), (np.float32, True), (np.float64, False)])
def test_emulation_matches_live_reference(reference, rs, cs, dtype, sorted_input):
    rescale_matrix, _, ScaledSVD, SVDModel = reference
    shape = (300, 90)
    idx, val = se.feedback_case(int(rs * 10 + cs * 100) + 1000, *shape, dtype=dtype, sorted_input=sorted_input)
    data = StubData(shape, train=(idx, val))
    base = SVDModel(data).get_training_matrix()
    model = ScaledSVD(data)
    model.row_scaling, model.col_scaling = rs, cs
    mats = [base, rescale_matrix(base, rs, 1), model.get_training_matrix()]
    for m in mats:
        m.sort_indices()
    check_against(*mats, idx, val, shape, rs, cs)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_downvote_emulation_matches_live_reference(reference, dtype):
    RecommenderModel = reference[1]
    rng = np.random.default_rng(5)
    s = rng.standard_normal((40, 300)).astype(dtype)
    rows, cols = rng.integers(0, 40, 2000), rng.integers(0, 300, 2000)
    low = s.copy()
    RecommenderModel.downvote_seen_items(low, (rows, cols))
    assert np.array_equal(se.reference_downvote(s, rows, cols).view(np.uint8), low.view(np.uint8))

"""HybridSVD on the host: the CHOLMOD stand-in (oracle/cholmod_stub.py), the f64 restatement against the recorded
reference runs (tests/golden/hybrid_cases.npz, made by oracle/make_hybrid_golden.py) and the host side of the device
model -- the ``(L, perm)`` -> K adapter and the float64 item projectors."""
import numpy as np
import pytest
import scipy.sparse as sps

from oracle import cholmod_stub
from oracle import hybrid_oracle as ho
from oracle import polara_oracle as po
from tests.helpers import subspace_gap


@pytest.fixture(scope="module")
def g(golden):
    return golden("hybrid_cases")


def _cases():
    from tests.conftest import load_golden
    return [str(c) for c in load_golden("hybrid_cases")["cases"]]


def _spd_similarity(n, seed):
    rng = np.random.default_rng(seed)
    f = sps.random(n, 12, density=0.15, random_state=seed, format="csr") + sps.eye(n, 12, format="csr")
    norm = np.sqrt(np.asarray(f.multiply(f).sum(1)).ravel())
    f = sps.diags(1.0 / np.maximum(norm, 1e-300)) @ f             # rows without features stay empty
    return (f @ f.T).tocsr(), rng


@pytest.mark.parametrize("beta", [1.0, 1.0 / 9.0])
def test_stub_factor_and_its_operations(beta):
    """L L^T = P (S + beta I) P^T, so K K^T = S + beta I for K = P^T L; dot / T.dot / T.solve are K v, K^T v, K^-T v."""
    s, rng = _spd_similarity(60, 3)
    f = cholmod_stub.cholesky(s, beta=beta)
    p = f.P()
    assert not np.array_equal(p, np.arange(60))                    # a real fill-reducing permutation
    low = f.L().toarray()
    assert np.allclose(np.triu(low, 1), 0.0)
    target = s.toarray() + beta * np.eye(60)
    np.testing.assert_allclose(low @ low.T, target[np.ix_(p, p)], atol=1e-12, rtol=0)
    k = ho.k_matrix(f)
    np.testing.assert_allclose(k @ k.T, target, atol=1e-12, rtol=0)
    v = rng.standard_normal((60, 5))
    np.testing.assert_array_equal(f.apply_P(v), v[p])
    np.testing.assert_array_equal(f.apply_Pt(f.apply_P(v)), v)
    np.testing.assert_allclose(f.apply_Pt(low @ v), k @ v, atol=1e-13)                     # chol.dot
    np.testing.assert_allclose(low.T @ f.apply_P(v), k.T @ v, atol=1e-13)                 # chol.T.dot
    np.testing.assert_allclose(f.apply_Pt(f.solve_Lt(v, use_LDLt_decomposition=False)),   # chol.T.solve
                               np.linalg.solve(k.T, v), atol=1e-10)
    sp_v = sps.random(60, 7, density=0.3, random_state=1, format="csr")
    np.testing.assert_allclose(f.apply_P(sp_v).toarray(), sp_v.toarray()[p])
    with pytest.raises(NotImplementedError):
        f.solve_Lt(v)


def test_stub_through_polaras_cholesky_factor():
    """polara's own CholeskyFactor (lib/cholesky.py) over the stub: the table of the reference calls."""
    from oracle import ref_driver as rd
    if rd.reference_root() is None:
        pytest.skip("reference not installed (oracle/_ref)")
    rd.import_reference()
    from polara.lib.cholesky import CholeskyFactor
    s, rng = _spd_similarity(40, 5)
    cf = CholeskyFactor(cholmod_stub.cholesky(s, beta=0.25))
    k = ho.k_matrix(cf._factor)
    v = rng.standard_normal((40, 3))
    np.testing.assert_allclose(cf.dot(v), k @ v, atol=1e-13)
    np.testing.assert_allclose(cf.T.dot(v), k.T @ v, atol=1e-13)
    np.testing.assert_allclose(cf.T.solve(v), np.linalg.solve(k.T, v), atol=1e-10)
    # the device model's host adapter reads the same factor
    from polara_b200.models import cholesky_factor_parts, cholesky_operator, hybrid_item_projectors
    low, perm = cholesky_factor_parts(cf)
    np.testing.assert_array_equal(perm, cf._factor.P())
    np.testing.assert_allclose(cholesky_operator(low, perm).toarray(), k, atol=0, rtol=0)
    left, right = hybrid_item_projectors(low, perm, v)
    np.testing.assert_allclose(left, cf.T.solve(v), atol=1e-11, rtol=1e-11)
    np.testing.assert_allclose(right, cf.dot(v), atol=1e-13, rtol=1e-13)


def test_host_adapter_from_an_l_perm_pair():
    """an ``(L, perm)`` pair gives the same K and projectors as the f64 oracle; a bad pair is refused."""
    from polara_b200.models import cholesky_factor_parts, cholesky_operator, hybrid_item_projectors
    s, rng = _spd_similarity(50, 7)
    f = cholmod_stub.cholesky(s, beta=0.5)
    low, perm = cholesky_factor_parts((f.L(), f.P()))
    assert sps.isspmatrix_csr(low) and low.dtype == np.float64 and perm.dtype == np.int64
    k = cholesky_operator(low, perm)
    np.testing.assert_allclose(k.toarray(), ho.k_matrix(f), atol=0, rtol=0)
    v = rng.standard_normal((50, 4))
    left, right = hybrid_item_projectors(low, perm, v)
    ref_left, ref_right = ho.projectors(f, v)
    np.testing.assert_allclose(left, ref_left, rtol=1e-11, atol=1e-12)
    np.testing.assert_allclose(right, ref_right, rtol=1e-13, atol=1e-14)
    # dropping the permutation changes the projectors: P is really applied
    left_id, right_id = hybrid_item_projectors(low, np.arange(50), v)
    assert not np.allclose(right_id, right)
    assert cholesky_factor_parts(None) is None
    with pytest.raises(ValueError):
        cholesky_factor_parts((f.L(), np.zeros(50, np.int64)))
    with pytest.raises(ValueError):
        cholesky_factor_parts((f.L()[:, :49], f.P()))


@pytest.mark.parametrize("name", _cases())
def test_oracle_reproduces_the_reference_runs(g, name):
    """svds of the explicit f64 operator K_u^T A K_i reproduces the reference's matrix-free (and precomputed) builds;
    the f64 projectors of its item factors and the lists they score reproduce the recorded ones."""
    c = ho.case(g, name)
    fi, fu = ho.factor(c, "item"), ho.factor(c, "user")
    np.testing.assert_array_equal(fi.P(), c["item_perm"])
    if fu is not None:
        np.testing.assert_array_equal(fu.P(), c["user_perm"])
    a = ho.training_matrix(c)
    op = ho.operator(a, ho.k_matrix(fi), None if fu is None else ho.k_matrix(fu))
    rank = int(c["rank"])
    v, s, _ = po.svd_build(sps.csr_matrix(op), rank)
    np.testing.assert_allclose(s, c["singular_values"], rtol=1e-9)
    assert subspace_gap(v, c["item_factors"]) < 1e-6
    left, right = ho.projectors(fi, c["item_factors"])
    np.testing.assert_allclose(left, c["projector_left"], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(right, c["projector_right"], rtol=1e-9, atol=1e-12)
    recs, _ = ho.recommend(c, c["projector_left"], c["projector_right"], int(c["topk"]))
    assert (recs == c["recs"]).mean() > 0.999
    # the host adapter of the device model gives the same projectors from (L, perm)
    from polara_b200.models import hybrid_item_projectors
    left_h, right_h = hybrid_item_projectors(sps.csr_matrix(fi.L()), fi.P(), c["item_factors"])
    np.testing.assert_allclose(left_h, c["projector_left"], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(right_h, c["projector_right"], rtol=1e-9, atol=1e-12)


def test_precomputed_and_matrix_free_runs_agree(g):
    """the reference's two branches of HybridSVD.build factorise the same operator."""
    for free, pre in (("both_w05", "both_w05_pre"),):
        a, b = ho.case(g, free), ho.case(g, pre)
        np.testing.assert_allclose(a["singular_values"], b["singular_values"], rtol=1e-9)
        assert subspace_gap(a["item_factors"], b["item_factors"]) < 1e-6

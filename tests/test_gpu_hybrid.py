"""HybridSVD on the device: the matrix-free factored operator K_u^T A K_i (pb200_rsvd_factored, Engine.rsvd with
factors, B200HybridSVD / B200ScaledHybridSVD, dropin_hybrid) against the plain build, an explicit f64 operator, the
recorded reference runs (tests/golden/hybrid_cases.npz) and polara's own HybridSVD on the CHOLMOD stand-in.  H100 only."""
import numpy as np
import pytest
import scipy.sparse as sps

from oracle import cholmod_stub
from oracle import hybrid_oracle as ho
from tests.helpers import check_topk_against_scores, subspace_gap

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    return get_engine()


def _similarity(n, n_features, seed):
    """cosine similarity of two sparse non-negative features per row (PSD, unit diagonal)."""
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(n), 2)
    cols = np.concatenate([rng.choice(n_features, 2, replace=False) for _ in range(n)])
    f = sps.csr_matrix((rng.random(len(rows)) + 0.5, (rows, cols)), shape=(n, n_features))
    f = sps.diags(1.0 / np.sqrt(np.asarray(f.multiply(f).sum(1)).ravel())) @ f
    return (f @ f.T).tocsr()


def _setup(m=900, n=500, per_user=30, seed=5):
    """planted ratings plus stub factors of an item (beta 1) and a user (beta 0.25) similarity matrix."""
    from polara_b200.synth import planted_ratings
    u, i, r = planted_ratings(m, n, per_user, rank=8, seed=seed)
    a = sps.csr_matrix((r.astype(np.float64), (u, i)), shape=(m, n))
    a.sum_duplicates()
    fi = cholmod_stub.cholesky(_similarity(n, max(8, n // 5), seed + 1), beta=1.0)
    fu = cholmod_stub.cholesky(_similarity(m, max(8, m // 5), seed + 2), beta=0.25)
    return u, i, r, a, fi, fu


def _data(u, i, r, shape):
    from polara_b200.host import ArrayData
    order = np.lexsort((i, u))
    return ArrayData(np.stack([u, i], axis=1), r, shape, test_user=u[order], test_item=i[order], test_fdbk=r[order],
                     test_shape=shape)


def _hybrid(data, rank, items=None, users=None, scaled=False, iters=40):
    from polara_b200.models import B200HybridSVD, B200ScaledHybridSVD
    model = (B200ScaledHybridSVD if scaled else B200HybridSVD)(data)
    model.verbose = False
    model.rank = rank
    model.power_iters = iters
    model.item_cholesky_factor = None if items is None else (items.L(), items.P())
    model.user_cholesky_factor = None if users is None else (users.L(), users.P())
    return model


def test_identity_factors_are_bit_equal_to_the_plain_build():
    """L = I, p = id: every SpMM of the chain copies its operand exactly, so factors and singular values (and U) are
    the plain build's bits; the projectors are then V itself."""
    from polara_b200.models import B200SVDModel
    u, i, r, a, _, _ = _setup()
    data = _data(u, i, r, a.shape)
    plain = B200SVDModel(data)
    plain.verbose = False
    plain.rank = 6
    plain.build(return_factors=True)
    eye_i = (sps.identity(a.shape[1], format="csr"), np.arange(a.shape[1]))
    eye_u = (sps.identity(a.shape[0], format="csr"), np.arange(a.shape[0]))
    model = _hybrid(data, 6, iters=plain.power_iters)
    model.item_cholesky_factor, model.user_cholesky_factor = eye_i, eye_u
    model.build(return_factors=True)
    for key in ("itemid", "userid", "singular_values"):
        np.testing.assert_array_equal(model.factors[key], plain.factors[key], err_msg=key)
    np.testing.assert_array_equal(model.factors["itemid_projector_left"], plain.factors["itemid"])
    np.testing.assert_array_equal(model.factors["itemid_projector_right"], plain.factors["itemid"])
    assert model.last_timings["subspace_iters"] == plain.last_timings["subspace_iters"]


def _check_against_explicit(model, a, ki, ku, rank, want_u):
    """matrix-free factors against svds of the explicit f64 operator and against that operator's Ritz residuals."""
    from oracle import polara_oracle as po
    op = ho.operator(a, ki, ku)
    v_ref, s_ref, _ = po.svd_build(sps.csr_matrix(op), rank)
    s = model.factors["singular_values"]
    v = model.factors["itemid"]
    np.testing.assert_allclose(s, s_ref, rtol=2e-4)
    assert subspace_gap(v, v_ref) <= 1e-2
    np.testing.assert_allclose(np.linalg.norm(op @ v, axis=0), s, rtol=1e-3)       # Ritz values of the operator
    if want_u:
        uu = model.factors["userid"]
        assert uu.shape == (a.shape[0], rank)
        # DESIGN.md section 4, rsvd with factors: ||M v_j - sigma_j u_j|| <= 2^-16 sigma_1 (three chained SpMMs) ...
        assert np.linalg.norm(op @ v - uu * s, axis=0).max() <= 2.0 ** -16 * s[0]
        # ... and ||M^T u_j - sigma_j v_j|| within the convergence tolerance
        assert np.linalg.norm(op.T @ uu - v * s, axis=0).max() <= 5e-3 * s[0]
        np.testing.assert_allclose(uu.T @ uu, np.eye(rank), atol=1e-4)


@pytest.mark.parametrize("sides", ["item", "user", "both"])
@pytest.mark.parametrize("want_u", [False, True])
def test_matrix_free_against_the_explicit_operator(sides, want_u):
    u, i, r, a, fi, fu = _setup()
    items = fi if sides in ("item", "both") else None
    users = fu if sides in ("user", "both") else None
    model = _hybrid(_data(u, i, r, a.shape), 3, items, users)
    model.build(return_factors=True if want_u else "vh")
    _check_against_explicit(model, a, None if items is None else ho.k_matrix(fi), None if users is None else ho.k_matrix(fu),
                            3, want_u)
    if items is not None:
        left, right = ho.projectors(fi, model.factors["itemid"])
        np.testing.assert_allclose(model.factors["itemid_projector_left"], left, rtol=1e-10, atol=1e-12)
        np.testing.assert_allclose(model.factors["itemid_projector_right"], right, rtol=1e-10, atol=1e-12)
    else:
        assert "itemid_projector_left" not in model.factors


def test_panel_major_factors(monkeypatch, eng):
    """a lowered L2 budget sends A, A^T and both factors panel-major (several column panels each)."""
    from polara_b200.engine import Engine
    monkeypatch.setattr(Engine, "PANEL_BYTES", 1 << 16)
    u, i, r, a, fi, fu = _setup(m=3000, n=1500, per_user=20, seed=9)
    assert eng.panel_cols_for(a.shape[0], 32) < a.shape[0] and eng.panel_cols_for(a.shape[1], 32) < a.shape[1]
    model = _hybrid(_data(u, i, r, a.shape), 3, fi, fu)
    model.build(return_factors=True)
    assert min(model.last_timings["panels"]) > 1
    _check_against_explicit(model, a, ho.k_matrix(fi), ho.k_matrix(fu), 3, True)


def test_second_build_gives_the_same_bits():
    u, i, r, a, fi, fu = _setup()
    model = _hybrid(_data(u, i, r, a.shape), 5, fi, fu)
    model.build(return_factors=True)
    first = {k: np.array(v) for k, v in model.factors.items()}
    model.build(return_factors=True)
    for key, val in first.items():
        np.testing.assert_array_equal(model.factors[key], val, err_msg=key)


def test_precomputed_operator_matches_matrix_free():
    """precompute_auxiliary_matrix: the explicit product formed by scipy and factorised as an operator."""
    u, i, r, a, fi, fu = _setup()
    free = _hybrid(_data(u, i, r, a.shape), 3, fi, fu)
    free.build()
    pre = _hybrid(_data(u, i, r, a.shape), 3, fi, fu)
    pre.precompute_auxiliary_matrix = True
    pre.build()
    np.testing.assert_allclose(pre.factors["singular_values"], free.factors["singular_values"], rtol=2e-4)
    assert subspace_gap(pre.factors["itemid"], free.factors["itemid"]) <= 1e-2


def _cases():
    from tests.conftest import load_golden
    return [str(c) for c in load_golden("hybrid_cases")["cases"]]


@pytest.mark.parametrize("name", _cases())
def test_model_reproduces_the_reference_runs(golden, name):
    """B200HybridSVD / B200ScaledHybridSVD on the recorded reference runs: sigma, subspace, >= 97 % list agreement
    paired with the tie-aware validity check on the model's own projectors, and evaluate() hit counts."""
    from polara_b200.host import ArrayData
    c = ho.case(golden("hybrid_cases"), name)
    fi, fu = ho.factor(c, "item"), ho.factor(c, "user")
    model = _hybrid(ArrayData.from_golden(c), int(c["rank"]), fi, fu, scaled=bool(c["scaled"]), iters=12)
    model.precompute_auxiliary_matrix = bool(c["precompute"])
    if bool(c["scaled"]):
        model.col_scaling, model.row_scaling = float(c["col_scaling"]), float(c["row_scaling"])
    model.build()
    np.testing.assert_allclose(model.factors["singular_values"], c["singular_values"], rtol=2e-4)
    assert subspace_gap(model.factors["itemid"], c["item_factors"]) < 2e-2
    recs = model.get_recommendations()
    assert recs.shape == c["recs"].shape and recs.dtype == np.int64
    assert (recs == c["recs"]).mean() > 0.97
    vl, vr = model.factors["itemid_projector_left"], model.factors["itemid_projector_right"]
    _, scores = ho.recommend(c, vl, vr, int(c["topk"]))
    shape = tuple(c["test_shape"])
    p = sps.csr_matrix((c["test_fdbk"].astype(np.float64), (c["test_user"], c["test_item"])), shape=shape)
    own = np.asarray(p.dot(vr)).dot(vl.T)
    tol = 4e-6 * np.abs(np.asarray(p.dot(vr))).sum(1).max() * np.abs(vl).max()
    assert check_topk_against_scores(recs, own, c["test_user"], c["test_item"], int(c["topk"]), tol) > 0.99
    hits = model.evaluate("hits")
    assert abs(hits.true_positive - c["hits"][0]) <= 3
    assert abs(hits.false_negative - c["hits"][3]) <= 3


def test_find_optimal_svd_rank_on_the_hybrid_model(golden):
    """the rank search sweeps through the right item projector, truncated with the factors at every rank."""
    from polara_b200.host import ArrayData
    from polara_b200.pipelines import find_optimal_svd_rank
    c = ho.case(golden("hybrid_cases"), "both_w05")
    model = _hybrid(ArrayData.from_golden(c), 12, ho.factor(c, "item"), ho.factor(c, "user"))
    model.build()
    ranks = [4, 8, 12]
    best, scores = find_optimal_svd_rank(model, ranks, "recall", return_scores=True)
    assert model.factors["itemid_projector_left"].shape[1] == 12             # factors protected
    full = dict(model.factors)
    for rank in ranks:
        model.rank = rank                                                     # truncation, no rebuild
        assert model._is_ready and model.factors["itemid_projector_right"].shape[1] == rank
        model._recommendations = None
        recall = model.evaluate("relevance").recall
        assert abs(recall - scores.loc[rank]) <= 0.01, rank
        model._rank, model.factors = 12, dict(full)
    assert best in ranks


def test_error_cases(eng):
    """mismatched factor shapes are refused (ValueError); factors under a reduce hook are not implemented."""
    from polara_b200.models import default_ell
    u, i, r, a, fi, fu = _setup(m=300, n=200, per_user=15)
    a_dev = eng.upload_csr(a.indptr.astype(np.int64), a.indices.astype(np.int32), a.data.astype(np.float32), a.shape)
    at_dev = eng.transpose(a_dev)

    def pair(k):
        k = sps.csr_matrix(k)
        d = eng.upload_csr(k.indptr.astype(np.int64), k.indices.astype(np.int32), k.data.astype(np.float32), k.shape)
        return d, eng.transpose(d)
    ell = default_ell(3)
    ki, ku = pair(ho.k_matrix(fi)), pair(ho.k_matrix(fu))
    with pytest.raises(ValueError):
        eng.rsvd(a_dev, at_dev, 3, ell, item_factor=ku)                      # user-sized factor on the item side
    with pytest.raises(ValueError):
        eng.rsvd(a_dev, at_dev, 3, ell, user_factor=ki)
    with pytest.raises(ValueError):
        eng.rsvd(a_dev, at_dev, 3, ell, item_factor=(ki[0], ku[1]))          # K and K^T of different factors
    eng.set_reduce_hook(lambda t: None)
    try:
        with pytest.raises(NotImplementedError):
            eng.rsvd(a_dev, at_dev, 3, ell, item_factor=ki)
    finally:
        eng.set_reduce_hook(None)
    v, s, _, _ = eng.rsvd(a_dev, at_dev, 3, ell, max_iters=30, item_factor=ki, user_factor=ku)   # the context still works
    assert np.isfinite(s.cpu().numpy()).all()


def test_dropin_matches_polaras_own_hybrid_svd():
    """dropin_hybrid(): the device build on polara's HybridSVD / ScaledHybridSVD against polara's own build, both on the
    CHOLMOD stand-in, on one SimilarityDataModel."""
    from oracle import ref_driver as rd
    if rd.reference_root() is None:
        pytest.skip("reference not installed (oracle/_ref)")
    rd.import_reference()
    import polara.recommender.hybrid.models as hm
    from oracle.make_hybrid_golden import make_data, similarity
    from polara_b200.models import dropin_hybrid
    from polara_b200.synth import planted_ratings
    old = getattr(hm, "cholesky_decomp_sparse", None)
    hm.cholesky_decomp_sparse = cholmod_stub.cholesky
    try:
        u, i, r = planted_ratings(600, 250, 25, rank=6, seed=21)
        cfg = dict(item_sim=similarity(250, 50, 2, 22), user_sim=similarity(600, 100, 2, 23))
        for ref_cls, mine_cls in zip((hm.HybridSVD, hm.ScaledHybridSVD), dropin_hybrid()):
            data = make_data((u, i, r), cfg)
            models = []
            for cls in (ref_cls, mine_cls):
                model = cls(data)
                model._sparse_mode = True
                model.verbose = False
                model.rank = 8
                model.features_weight = 0.7
                model.build()
                models.append(model)
            ref, mine = models
            np.testing.assert_allclose(mine.factors["singular_values"], ref.factors["singular_values"], rtol=2e-4)
            assert subspace_gap(mine.factors["itemid"], ref.factors["itemid"]) < 2e-2
            ref_recs, recs = ref.get_recommendations(), mine.get_recommendations()
            assert recs.shape == ref_recs.shape and (recs == ref_recs).mean() > 0.97
            h_ref, h_mine = ref.evaluate("hits"), mine.evaluate("hits")
            assert abs(h_ref.true_positive - h_mine.true_positive) <= 3
            assert mine.item_cholesky_factor._L is None                        # _clear_cholesky_cache ran
    finally:
        hm.cholesky_decomp_sparse = old

"""Oracle vs outputs of the reference (evfro/polara) itself, recorded by oracle/make_golden.py into
tests/golden/reference_live.npz together with the inputs the reference's data model handed over.  CPU only."""
import numpy as np
import pytest
import scipy.sparse as sps

from oracle import polara_oracle as po


@pytest.fixture(scope="module")
def ref(golden):
    return golden("reference_live")


@pytest.mark.parametrize("seed", [1, 2])
def test_downvote_topk_rescale_live(ref, seed):
    rng = np.random.default_rng(seed)
    s = rng.standard_normal((20, 50))
    rows = np.repeat(np.arange(20), 4)
    cols = np.concatenate([rng.choice(50, 4, replace=False) for _ in range(20)])
    mine = po.downvote_seen_items(s.copy(), rows, cols)
    np.testing.assert_array_equal(mine, ref["dv%d_downvoted" % seed])
    for row in range(20):
        np.testing.assert_array_equal(po.topsort(mine[row], 6), ref["dv%d_topsort6" % seed][row])
    a = sps.random(40, 30, density=0.2, random_state=seed, format="csr")
    for j, (scaling, axis) in enumerate(((0.4, 0), (0.8, 1), (1, 0))):
        np.testing.assert_allclose(po.rescale_matrix(a, scaling, axis).toarray(), ref["dv%d_rescaled%d" % (seed, j)],
                                   rtol=1e-14)


def test_hooi_live(ref):
    rng = np.random.default_rng(3)
    shp = (40, 30, 5)
    nnz = 900
    idx = np.unique(np.stack([rng.integers(0, s, nnz) for s in shp], axis=1), axis=0).astype(np.intp)
    val = np.ones(len(idx))
    mine = po.hooi(idx, val, shp, (4, 3, 2), num_iters=6, growth_tol=1e-4, seed=5)
    for j in range(3):
        sv = np.linalg.svd(mine[j].T @ ref["hooi_f%d" % j], compute_uv=False)
        assert sv.min() > 1 - 1e-9
    np.testing.assert_allclose(np.linalg.norm(mine[3]), np.linalg.norm(ref["hooi_core"]), rtol=1e-10)


def test_c1_shaped_svd_model_live(ref):
    """PureSVD rank 10, top-10 at ML-1M density (1200 x 740 users x items, 166 ratings per user) through the reference's
    RecommenderData.prepare + SVDModel.build + get_recommendations, against the oracle on the arrays the reference's data
    model handed over: singular values, item-factor subspace, and every recommendation list (scored with the reference's
    own factors: exact; with the oracle's factors: up to near-ties)."""
    idx, val, shp = ref["svd_train_idx"], ref["svd_train_val"].astype(np.float64), tuple(ref["svd_train_shape"])
    recs = ref["svd_recs"]
    a = sps.csr_matrix((val, (idx[:, 0], idx[:, 1])), shape=shp, dtype=np.float64)
    v, s, _ = po.svd_build(a, 10)
    np.testing.assert_allclose(s, ref["svd_sigma"], rtol=1e-9)
    vref = ref["svd_v"]
    assert np.linalg.svd(v.T @ vref, compute_uv=False).min() > 1 - 1e-6
    tu, ti, tf = ref["svd_test_u"], ref["svd_test_i"], ref["svd_test_f"].astype(np.float64)
    tshape = tuple(ref["svd_test_shape"])
    mine = po.recommend_svd(tu, ti, tf, tshape, vref, topk=10)
    assert mine.shape == recs.shape and recs.shape[1] == 10
    np.testing.assert_array_equal(mine, recs)
    own = po.recommend_svd(tu, ti, tf, tshape, v, topk=10)
    assert (own == recs).mean() > 0.99


def test_coffee_model_live_default_mlrank(ref):
    """CoffeeModel with the reference's default multilinear rank (13, 10, 2) on a 1500 x 600 x 5 tensor through the
    reference against the oracle: HOOI from the same seed (factor subspaces, core norm) and every recommendation list
    scored with the reference's factors."""
    idx, val, shp = ref["cf_train_idx"].astype(np.intp), ref["cf_train_val"].astype(np.float64), tuple(ref["cf_train_shape"])
    assert tuple(ref["cf_mlrank"]) == (13, 10, 2)
    mine = po.hooi(idx, val, shp, tuple(int(x) for x in ref["cf_mlrank"]), num_iters=int(ref["cf_num_iters"]),
                   growth_tol=float(ref["cf_growth_tol"]), seed=int(ref["cf_seed"]))
    for j in range(3):
        assert np.linalg.svd(mine[j].T @ ref["cf_f%d" % j], compute_uv=False).min() > 1 - 1e-6, j
    np.testing.assert_allclose(np.linalg.norm(mine[3]), np.linalg.norm(ref["cf_core"]), rtol=1e-8)
    tu, ti, tf = ref["cf_test_u"], ref["cf_test_i"], ref["cf_test_f"]
    lists = po.recommend_coffee(tu, ti, tf, tuple(ref["cf_test_shape"]), ref["cf_f1"], ref["cf_f2"], topk=10)
    np.testing.assert_array_equal(lists, ref["cf_recs"])


def test_round_core_live(ref):
    """CoffeeModel.round_core / _check_reduced_rank (models.py:949-980) against the oracle restatement."""
    core = ref["rc_core"]
    np.testing.assert_array_equal(core, np.random.default_rng(9).standard_normal((7, 6, 4)))
    for j, (mode, rank) in enumerate(((0, 3), (1, 6), (1, 2), (2, 1), (2, 3))):
        rot, new_core = po.round_core(core, mode, rank)
        np.testing.assert_allclose(rot, ref["rc%d_rot" % j], rtol=0, atol=1e-13)
        np.testing.assert_allclose(new_core, ref["rc%d_core" % j], rtol=0, atol=1e-13)
        assert new_core.shape[mode] == rank


@pytest.mark.parametrize("switch_positive", [None, 4])
def test_simple_rates_match_reference_live(ref, switch_positive):
    """evaluate(simple_rates=True) / holdout_size == 1 (models.py:451-458): hit rate, ARHR and MRR of the host mirror
    against the reference's own evaluation functions on random lists."""
    from polara_b200.host import evaluate_lists
    rng = np.random.default_rng(12)
    m, n, k = 60, 90, 10
    recs = np.stack([rng.choice(n, k, replace=False) for _ in range(m)])
    hu = np.repeat(np.arange(m), 3)
    hi = np.concatenate([rng.choice(n, 3, replace=False) for _ in range(m)])
    hf = rng.integers(1, 6, size=len(hu)).astype(np.float64)
    rel, rank = evaluate_lists(recs, hu, hi, hf, n, metric_type=["relevance", "ranking"], switch_positive=switch_positive,
                               simple_rates=True)
    hr_ref, arhr_ref, mrr_ref = ref["rates_%s" % switch_positive]
    np.testing.assert_allclose(rel.hr, hr_ref, rtol=1e-12)
    np.testing.assert_allclose(rank.arhr, arhr_ref, rtol=1e-12)
    np.testing.assert_allclose(rank.mrr, mrr_ref, rtol=1e-12)

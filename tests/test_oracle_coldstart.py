"""Item cold start on the host side: the f64 oracle (oracle/coldstart_oracle.py) against the recorded reference runs
(tests/golden/coldstart_cases.npz), the stand-alone data model's ordering and dropping rules (host.ColdStartData), and
``evaluate()`` along the cold-item axis.  CPU only."""
import numpy as np
import pytest
import scipy.sparse as sps

from oracle import coldstart_oracle as co


def _cases():
    from tests.conftest import load_golden
    return [str(c) for c in load_golden("coldstart_cases")["cases"]]


@pytest.mark.parametrize("name", _cases())
def test_oracle_reproduces_the_reference_runs(golden, name):
    """W, its transform and the lists from the recorded factors, at the built rank and at the lower one."""
    c = co.case(golden("coldstart_cases"), name)
    f, f_cold = co.csr(c, "F"), co.csr(c, "F_cold")
    assert f.shape[0] == c["train_shape"][1] and f_cold.shape == (len(c["cold_new"]), f.shape[1])
    w = co.feature_mapping(f, co.mapping_source(c))
    np.testing.assert_allclose(w, c["W"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(co.transform(w), c["transform"], rtol=1e-9, atol=1e-12 * np.abs(c["transform"]).max())
    recs, _ = co.recommend(f_cold, c["W"], c["transform"], c["user_factors"], c["singular_values"], int(c["topk"]))
    np.testing.assert_array_equal(recs, c["recs"])
    u, s, w_low, t_low = co.truncated(c, int(c["low_rank"]))
    np.testing.assert_allclose(t_low, c["transform_low"], rtol=1e-9, atol=1e-12 * np.abs(t_low).max())
    recs_low, _ = co.recommend(f_cold, w_low, t_low, u, s, int(c["topk"]))
    np.testing.assert_array_equal(recs_low, c["recs_low"])


# evaluate('all'): relevance (precision, recall, fallout, specifity, miss_rate), ranking (ndcg, ndcl, map, arhr),
# experience (coverage), hits (tp, fp, tn, fn).  ndcg / ndcl are never compared: the reference leaves masked entries
# of safe_divide uninitialised.
COMPARED = {0: "precision", 1: "recall", 4: "miss_rate", 7: "map", 8: "arhr", 9: "coverage", 10: "tp", 11: "fp",
            13: "fn"}


def _flat(res):
    return np.array([np.nan if x is None else float(x) for t in res for x in t])


def _model_with_lists(data, recs):
    from polara_b200.models import B200SVDModelItemColdStart
    model = B200SVDModelItemColdStart(data)
    model.verbose = False
    model.topk = recs.shape[1]
    model._recommendations = np.asarray(recs)
    model._is_ready = True
    return model


@pytest.mark.parametrize("name", _cases())
def test_evaluate_on_the_cold_axis_matches_the_reference(golden, name):
    """the reference's lists through ``evaluate()`` of the stand-alone model give the reference's recorded metrics, at
    both ranks."""
    c = co.case(golden("coldstart_cases"), name)
    for recs, ev in ((c["recs"], c["evaluate"]), (c["recs_low"], c["evaluate_low"])):
        got = _flat(_model_with_lists(co.data(c), recs).evaluate())
        for j, what in COMPARED.items():
            assert got[j] == pytest.approx(ev[j], rel=1e-12, abs=1e-15), what


def test_evaluate_against_a_hand_count():
    """3 cold items, 5 users, top-2.  Holdout pairs (cold item, user): item 0 -> users 1, 3; item 1 -> user 4;
    item 2 -> users 0, 2, 4."""
    from polara_b200.host import ColdStartData
    f = sps.csr_matrix(np.eye(4)[:3])                                # 3 training items, 4 features
    fc = sps.csr_matrix(np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0.]]))
    data = ColdStartData(np.array([[0, 0], [1, 1], [2, 2]]), np.ones(3), (5, 3), [2, 0, 1, 0, 2, 2], [0, 1, 4, 3, 2, 4],
                         np.ones(6), f, fc, n_users=5)
    recs = np.array([[1, 0], [2, 4], [4, 1]])                       # hits: (0,1)@1; (1,4)@2; (2,4)@1
    model = _model_with_lists(data, recs)
    hits = model.evaluate("hits")
    assert (hits.true_positive, hits.false_positive, hits.false_negative) == (3, 3, 3)
    rel = model.evaluate("relevance")
    assert rel.precision == pytest.approx(np.mean([1 / 2, 1 / 2, 1 / 2]))
    assert rel.recall == pytest.approx(np.mean([1 / 2, 1 / 1, 1 / 3]))
    ranking = model.evaluate("ranking")
    assert ranking.arhr == pytest.approx(np.mean([1, 1 / 2, 1]))
    assert ranking.map == pytest.approx(np.mean([1 / 2, (1 / 2) / 1, 1 / 2]))
    assert model.evaluate("experience").coverage == pytest.approx(4 / 5)      # users 0, 1, 2, 4 of 5


def test_data_orders_and_drops_as_the_reference():
    """holdout sorted by cold id (stable); a cold item without a feature any training item has is dropped with its
    rows; unknown features are dropped from F_cold; representative users filter the holdout only when some cold item
    has none of them."""
    from polara_b200.host import ColdStartData
    f = sps.csr_matrix(np.array([[1, 0, 0, 0, 0], [0, 1, 1, 0, 0], [1, 0, 0, 0, 0.]]))      # features 3, 4 unseen
    fc = sps.csr_matrix(np.array([[0, 0, 1, 1, 0],           # cold 0: feature 2 shared, 3 unknown
                                  [0, 0, 0, 1, 1],           # cold 1: unknown features only -> dropped
                                  [1, 0, 0, 0, 0],           # cold 2
                                  [0, 1, 0, 0, 0.]]))        # cold 3
    item = np.array([3, 1, 0, 2, 3, 0, 1, 2])
    user = np.array([5, 0, 2, 1, 0, 4, 3, 3])
    fdbk = np.arange(8.0)
    data = ColdStartData(np.array([[0, 0], [1, 1], [2, 2]]), np.ones(3), (6, 3), item, user, fdbk, f, fc, n_users=6)
    hold = data.test.holdout
    np.testing.assert_array_equal(hold["itemid_cold"].values, [0, 0, 2, 2, 3, 3])
    np.testing.assert_array_equal(hold["userid"].values, [2, 4, 1, 3, 5, 0])
    np.testing.assert_array_equal(hold["rating"].values, [2, 5, 3, 7, 0, 4])
    np.testing.assert_array_equal(data.index.itemid.cold_start, [0, 2, 3])
    np.testing.assert_array_equal(data.cold_item_features.toarray(),
                                  [[0, 0, 1, 0, 0], [1, 0, 0, 0, 0], [0, 1, 0, 0, 0]])
    assert data.index.userid.shape[0] == 6 and data.index.itemid.training.shape[0] == 3
    # representative users 1 and 4: cold 3 keeps no row and goes; cold 0 and 2 keep one row each
    data = ColdStartData(np.array([[0, 0], [1, 1], [2, 2]]), np.ones(3), (6, 3), item, user, fdbk, f, fc, n_users=6,
                         representative_users=[4, 1])
    np.testing.assert_array_equal(data.test.holdout["itemid_cold"].values, [0, 2])
    np.testing.assert_array_equal(data.test.holdout["userid"].values, [4, 1])
    np.testing.assert_array_equal(data.index.itemid.cold_start, [0, 2])
    assert data.cold_item_features.shape == (2, 5)
    # representative users 2, 1 and 0: every kept cold item has one, so the reference sets up no filter at all
    data = ColdStartData(np.array([[0, 0], [1, 1], [2, 2]]), np.ones(3), (6, 3), item, user, fdbk, f, fc, n_users=6,
                         representative_users=[2, 1, 0])
    np.testing.assert_array_equal(data.test.holdout["userid"].values, [2, 4, 1, 3, 5, 0])
    np.testing.assert_array_equal(data.index.itemid.cold_start, [0, 2, 3])
    with pytest.raises(ValueError):
        ColdStartData(np.array([[0, 0]]), np.ones(1), (6, 3), item, user, fdbk, f[:2], fc)


@pytest.mark.parametrize("name", _cases())
def test_data_rebuilds_the_recorded_split(golden, name):
    """the recorded holdout and F_cold, shuffled and joined by a cold item with unknown features only, come out of
    ColdStartData as the reference's post-processing left them."""
    from polara_b200.host import ColdStartData
    c = co.case(golden("coldstart_cases"), name)
    n_feat = int(c["F_shape"][1])
    n_cold = int(c["cold_new"].max()) + 2                              # one extra cold item at the end
    rows = np.zeros((n_cold, n_feat + 1))
    rows[c["cold_new"], :n_feat] = co.csr(c, "F_cold").toarray()
    rows[-1, n_feat] = 1.0                                             # a feature no training item has
    f = sps.hstack([co.csr(c, "F"), sps.csr_matrix((int(c["F_shape"][0]), 1))]).tocsr()
    rng = np.random.default_rng(0)
    item = np.r_[c["holdout_cold"], [n_cold - 1] * 3]
    user = np.r_[c["holdout_user"], [0, 1, 2]]
    fdbk = np.r_[c["holdout_fdbk"], [5.0] * 3]
    perm = rng.permutation(len(item))
    data = ColdStartData(c["train_idx"], c["train_val"], c["train_shape"], item[perm], user[perm], fdbk[perm], f,
                         sps.csr_matrix(rows), n_users=int(c["n_users"]))
    hold = data.test.holdout
    np.testing.assert_array_equal(hold["itemid_cold"].values, c["holdout_cold"])
    np.testing.assert_array_equal(data.index.itemid.cold_start, c["cold_new"])
    np.testing.assert_array_equal(data.cold_item_features[:, :n_feat].toarray(), co.csr(c, "F_cold").toarray())
    for cold in np.unique(c["holdout_cold"]):                          # the same (user, feedback) pairs per cold item
        mine = hold[hold["itemid_cold"] == cold]
        sel = c["holdout_cold"] == cold
        assert sorted(zip(mine["userid"], mine["rating"])) == sorted(zip(c["holdout_user"][sel], c["holdout_fdbk"][sel]))


def test_rank_change_truncates_w_and_recomputes_the_transform(golden):
    """the host side of a rank change on recorded factors: W is cut with the other factors, the transform is
    recomputed at the lower rank, and a rank above the built one clears the factors and the transform."""
    c = co.case(golden("coldstart_cases"), "svd")
    from polara_b200.models import B200SVDModelItemColdStart
    model = B200SVDModelItemColdStart(co.data(c))
    model.verbose = False
    rank = int(c["rank"])
    model._rank = rank
    model.factors = {"userid": c["user_factors"], "itemid": c["item_factors"], "singular_values": c["singular_values"],
                     "itemid_features": c["W"]}
    model._item_features_transform_helper = c["transform"]
    model._is_ready = True
    model.rank = int(c["low_rank"])
    assert model.item_features_embeddings.shape[1] == int(c["low_rank"])
    np.testing.assert_allclose(model._item_features_transform_helper, c["transform_low"], rtol=1e-9,
                               atol=1e-12 * np.abs(c["transform_low"]).max())
    model.rank = rank + 1
    assert not model._is_ready and model.item_features_embeddings is None
    assert model._item_features_transform_helper is None
    assert model._prediction_key == "itemid_cold" and model._prediction_target == "userid" and not model.filter_seen

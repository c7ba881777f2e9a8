"""The reference's rank search (find_optimal_svd_rank) recorded in tests/golden/rank_sweep.npz
(oracle/make_rank_sweep_golden.py) against the host restatements: the oracle reproduces the sampled lists at every
rank, host.evaluate_lists reproduces the metric series from the recorded lists, and polara_b200.pipelines'
find_optimal_svd_rank, fed the recorded lists by one sweep, returns the reference's best rank and scores."""
import os

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sps

from oracle import sampler_oracle as so
from tests.helpers import check_topk_against_scores

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rank_sweep.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def _profile(g, c):
    shape = tuple(int(x) for x in g[c + "shape"])
    tu, ti, tf = g[c + "test_user"], g[c + "test_item"], g[c + "test_fdbk"]
    keep = tf != 0
    return sps.csr_matrix((tf[keep], (tu[keep], ti[keep])), shape=shape), shape


def test_fixture_records_every_rank(g):
    for c, build_rank in (("s_", 12), ("k_", 16)):
        ranks = [int(r) for r in g[c + "ranks"]]
        assert max(ranks) == build_rank == g[c + "item_factors"].shape[1]
        assert len(g[c + "scores"]) == len(ranks)
        for r in ranks:
            assert g[c + "lists_r%d" % r].shape == (int(g[c + "shape"][0]), int(g[c + "topk"]))
    assert int(g["s_best"]) in [int(r) for r in g["s_ranks"]]


def test_oracle_reproduces_the_sampled_lists_at_every_rank(g):
    profile, shape = _profile(g, "s_")
    hu, hi = g["s_holdout_user"], g["s_holdout_item"]
    indptr, indices = so.exclusion_lists(profile, hu, hi, shape)
    seeds = np.random.SeedSequence(int(g["s_data_seed"])).generate_state(shape[0])
    drawn = so.sample_rows(indptr, indices, shape[1], int(g["s_n_unseen"]), seeds)
    v = g["s_item_factors"]
    k = int(g["s_topk"])
    for r in g["s_ranks"]:
        vr = v[:, :int(r)]
        e = profile.dot(vr)
        hold = np.einsum("ur,ur->u", e, vr[hi])[:, None]
        s64 = np.concatenate([hold, so.sampled_scores(e, vr, drawn)], axis=1)
        lists = g["s_lists_r%d" % r]
        exact = check_topk_against_scores(lists, s64, [], [], k, 1e-9 * np.abs(s64).max())
        assert exact >= 0.99, (int(r), exact)


def test_evaluate_lists_reproduces_the_recorded_series(g):
    from polara_b200.host import evaluate_lists
    for j, r in enumerate(g["s_ranks"]):
        got = evaluate_lists(g["s_lists_r%d" % r], g["s_holdout_user"], g["s_holdout_pos"], None, int(g["s_n_items"]),
                             metric_type="ranking", simple_rates=True)
        assert got.mrr == pytest.approx(g["s_scores"][j], rel=1e-12), int(r)
    for j, r in enumerate(g["k_ranks"]):
        got = evaluate_lists(g["k_lists_r%d" % r], g["k_holdout_user"], g["k_holdout_item"], g["k_holdout_fdbk"],
                             int(g["k_n_items"]), metric_type="relevance")
        assert got.recall == pytest.approx(g["k_scores"][j], rel=1e-12), int(r)


def stand_alone_model(g, c):
    """a stand-alone B200SVDModel on the fixture's test data with the reference's factors; the sampled case predicts
    holdout positions (``x_itemid``) from a data model that draws 99 unseen items on the fly, as the fixture's did."""
    from polara_b200.host import ArrayData
    from polara_b200.models import B200SVDModel
    shape = tuple(int(x) for x in g[c + "shape"])
    hold = pd.DataFrame({"userid": g[c + "holdout_user"], "itemid": g[c + "holdout_item"]})
    if c == "s_":
        hold["rating"] = np.ones(len(hold))
        hold["x_itemid"] = g["s_holdout_pos"]
    else:
        hold["rating"] = g["k_holdout_fdbk"]
    n_hold = len(hold) // shape[0]
    data = ArrayData(np.zeros((1, 2), dtype=np.int64), np.ones(1), (shape[0], int(g[c + "n_items"])),
                     g[c + "test_user"], g[c + "test_item"], g[c + "test_fdbk"], shape, holdout=hold, warm_start=False,
                     holdout_size=n_hold)
    model = B200SVDModel(data)
    model.verbose = False
    v = g[c + "item_factors"]
    model.rank = v.shape[1]
    model.topk = int(g[c + "topk"])
    model.factors = {"userid": None, "itemid": v, "singular_values": np.ones(v.shape[1])}
    model._is_ready = True
    if c == "s_":
        model._prediction_target = "x_itemid"
        data.unseen_interactions = None
        data.unseen_items_num = int(g["s_n_unseen"])
        data.seed = int(g["s_data_seed"])
    return model


@pytest.mark.parametrize("case", ["s_", "k_"])
def test_find_optimal_svd_rank_with_recorded_lists(g, case):
    from polara_b200 import pipelines
    model = stand_alone_model(g, case)
    ranks = [int(r) for r in g[case + "ranks"]]
    calls = []

    def sweep(*args, **kwargs):
        calls.append((args, kwargs))
        return {r: g[case + "lists_r%d" % r] for r in ranks}
    model.rank_sweep = sweep
    model.sampled_rank_sweep = sweep
    v = model.factors["itemid"]
    if case == "s_":
        target, kw = "mrr", dict(metric_type="ranking", simple_rates=True)
    else:
        target, kw = "recall", dict(metric_type="relevance")
    best, scores = pipelines.find_optimal_svd_rank(model, ranks, target, return_scores=True, **kw)
    assert len(calls) == 1
    if case == "s_":
        (sweep_ranks, holdout_items, unseen), kwargs = calls[0]
        assert unseen is None and kwargs["n_unseen"] == 99 and kwargs["seed"] == int(g["s_data_seed"])
        np.testing.assert_array_equal(holdout_items.ravel(), g["s_holdout_item"])
    assert best == int(g[case + "best"])
    # same index, name and order; values to the last bits: the reference averages the reciprocal ranks of an m x 1
    # matrix (a sequential sum), host.evaluate_lists a vector (numpy's pairwise sum)
    want = pd.Series(g[case + "scores"], index=pd.Index(ranks, name="rank"), name=model.method)
    pd.testing.assert_series_equal(scores, want, check_exact=False, rtol=1e-12, atol=0)
    assert model.factors["itemid"] is v and model._rank == max(ranks)
    assert model._recommendations is None


def test_find_optimal_svd_rank_rebuilds_and_restores(g):
    """a model that is not ready is built at max(max(ranks), model.rank); config is applied first."""
    from polara_b200 import pipelines
    model = stand_alone_model(g, "k_")
    model._is_ready = False
    built = []

    def build():
        built.append(model.rank)
        model._is_ready = True
    model.build = build
    model.rank_sweep = lambda ranks: {r: g["k_lists_r%d" % r] for r in ranks}
    best = pipelines.find_optimal_svd_rank(model, [12, 8], "recall", config={"topk": 10}, metric_type="relevance")
    assert built == [16] and best in (12, 8)
    assert model._rank == 16 and model.factors["itemid"].shape[1] == 16


def test_sweep_rank_limits_and_sharding(g):
    """ranks beyond the current factors would need a rebuild; item-sharded models have no sweep (no device needed:
    both are refused before any work)."""
    model = stand_alone_model(g, "k_")
    for sweep in (model.rank_sweep, lambda r: model.sampled_rank_sweep(r, np.zeros((120, 3)), n_unseen=9, seed=1)):
        with pytest.raises(ValueError, match="rebuild"):
            sweep([8, 17])
        with pytest.raises(ValueError, match="rebuild"):
            sweep([0, 8])
    model.shard = object()
    with pytest.raises(NotImplementedError, match="sharded"):
        model.rank_sweep([8])
    with pytest.raises(NotImplementedError, match="sharded"):
        model.sampled_rank_sweep([8], np.zeros((120, 3)), np.zeros((120, 5)))

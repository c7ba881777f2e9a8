"""The reference's Tucker-rank search (find_optimal_tucker_ranks) recorded in tests/golden/tucker_sweep.npz
(oracle/make_tucker_sweep_golden.py) against the host side of the device search: host.evaluate_lists reproduces the
recorded scores from the recorded lists, round_tucker_core reproduces the rounded factors of every triple, and
polara_b200.pipelines' find_optimal_tucker_ranks, fed the recorded lists by one sweep, visits the reference's triples in
its order and returns its best triple and Series.  No device: the sweep is stubbed, and its argument checks run first."""
import os

import numpy as np
import pandas as pd
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tucker_sweep.npz")
CASES = ("a_", "b_")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def case_arrays(g, c):
    return {k[len(c):]: g[k] for k in g.files if k.startswith(c)}


def key(t):
    return "%d_%d_%d" % tuple(t)


def visited(g, c):
    return [tuple(int(x) for x in t) for t in g[c + "visited"]]


def switch_positive(g, c):
    sp = float(g[c + "switch_positive"])
    return None if np.isnan(sp) else sp


def tucker_ranks(g, c):
    return [[int(x) for x in g[c + "ranks_r%d" % m]] for m in (1, 2, 3)]


def flattener(g, c):
    fl = g[c + "flattener"]
    return None if fl.ndim == 0 and int(fl) == -1 else [int(x) for x in np.atleast_1d(fl)]


def stand_alone_model(g, c, model_class=None):
    """a stand-alone B200CoffeeModel on the fixture's data with the reference's full-build factors, ready to score."""
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CoffeeModel
    a = case_arrays(g, c)
    model = (model_class or B200CoffeeModel)(ArrayData.from_golden(a))
    model.verbose = False
    model.topk = int(a["topk"])
    model.switch_positive = switch_positive(g, c)
    if flattener(g, c) is not None:
        model.flattener = flattener(g, c)
    model.factors = {"userid": a["u0"], "itemid": a["u1"], "rating": a["u2"], "core": a["core"]}
    model._mlrank = tuple(int(x) for x in a["mlrank"])
    model._is_ready = True
    return model


def test_fixture_records_every_visited_triple(g):
    for c in CASES:
        seen = visited(g, c)
        assert len(seen) == len(set(seen)) == len(g[c + "scores"])
        assert sorted(seen) == [tuple(int(x) for x in t) for t in g[c + "score_index"]]
        for t in seen:
            assert g[c + "lists_" + key(t)].shape == (int(g[c + "test_shape"][0]), int(g[c + "topk"]))
    # the grids exercise the skip rule (a_) and same_space (b_)
    assert (10, 2, 1) not in visited(g, "a_") and (2, 8, 1) not in visited(g, "a_")
    assert all(t[0] == t[1] for t in visited(g, "b_"))


def test_evaluate_lists_reproduces_the_recorded_series(g):
    from polara_b200.host import evaluate_lists
    for c in CASES:
        for t, want in zip(g[c + "score_index"], g[c + "scores"]):
            got = evaluate_lists(g[c + "lists_" + key(t)], g[c + "holdout_user"], g[c + "holdout_item"],
                                 g[c + "holdout_fdbk"], int(g[c + "n_items"]), metric_type="relevance",
                                 switch_positive=switch_positive(g, c))
            assert got.recall == pytest.approx(want, rel=1e-12), (c, tuple(t))


def test_host_rounding_reproduces_the_reference_factors(g):
    """``mlrank = t`` on the full build (models.py:949-980): modes 0, 1, 2 rounded in turn from the full core."""
    from polara_b200.models import round_tucker_core
    for c in CASES:
        full = [g[c + "u0"], g[c + "u1"], g[c + "u2"]]
        for t in visited(g, c):
            core, out = g[c + "core"], list(full)
            for mode in range(3):
                if full[mode].shape[1] > t[mode]:
                    rot, core = round_tucker_core(core, mode, t[mode])
                    out[mode] = full[mode].dot(rot)
            np.testing.assert_allclose(out[1], g[c + "item_" + key(t)], rtol=0, atol=1e-12, err_msg=str(t))
            np.testing.assert_allclose(out[2], g[c + "fdbk_" + key(t)], rtol=0, atol=1e-12, err_msg=str(t))


def _stub_sweep(g, c, model, calls):
    def sweep(mlranks):
        calls.append(list(mlranks))
        return {tuple(t): g[c + "lists_" + key(t)] for t in mlranks}
    model.tucker_rank_sweep = sweep


@pytest.mark.parametrize("c", CASES)
def test_find_optimal_tucker_ranks_with_recorded_lists(g, c):
    from polara_b200 import pipelines
    model = stand_alone_model(g, c)
    calls, order = [], []
    _stub_sweep(g, c, model, calls)
    full = dict(model.factors)
    full_rank = model._mlrank

    def evaluator(m, target_metric, **kw):
        order.append(m._mlrank)
        assert m.factors["itemid"] is full["itemid"] and m.factors["core"] is full["core"]
        np.testing.assert_array_equal(m.recommendations, g[c + "lists_" + key(m._mlrank)])
        return pipelines.evaluate_models(m, target_metric, **kw)
    best, scores = pipelines.find_optimal_tucker_ranks(model, tucker_ranks(g, c), "recall", return_scores=True,
                                                       same_space=bool(g[c + "same_space"]), evaluator=evaluator,
                                                       metric_type="relevance")
    assert order == visited(g, c)
    assert len(calls) == 1 and sorted(calls[0]) == sorted(visited(g, c))
    assert best == tuple(int(x) for x in g[c + "best"])
    idx = pd.MultiIndex.from_tuples([tuple(int(x) for x in t) for t in g[c + "score_index"]], names=["r1", "r2", "r3"])
    want = pd.Series(g[c + "scores"], index=idx, name=model.method)
    pd.testing.assert_series_equal(scores, want, check_exact=False, rtol=1e-12, atol=0)
    assert model._mlrank == full_rank and model.factors == full and model._recommendations is None
    assert model.verbose is False


def test_default_evaluator_and_restore_on_error(g):
    """without return_scores only the best triple comes back; when the evaluator raises, ``_mlrank`` and ``factors`` are
    restored (what the reference's ``finally`` restores)."""
    from polara_b200 import pipelines
    c = "a_"
    model = stand_alone_model(g, c)
    _stub_sweep(g, c, model, [])
    best = pipelines.find_optimal_tucker_ranks(model, tucker_ranks(g, c), "recall", metric_type="relevance")
    assert best == tuple(int(x) for x in g[c + "best"])
    full = dict(model.factors)
    full_rank = model._mlrank
    n = []

    def failing(m, target_metric, **kw):
        n.append(m._mlrank)
        if len(n) == 3:
            raise RuntimeError("evaluator failed")
        return pipelines.evaluate_models(m, target_metric, **kw)
    with pytest.raises(RuntimeError, match="evaluator failed"):
        pipelines.find_optimal_tucker_ranks(model, tucker_ranks(g, c), "recall", evaluator=failing,
                                            metric_type="relevance")
    assert n == visited(g, c)[:3]
    assert model._mlrank == full_rank and model.factors == full


def test_find_optimal_tucker_ranks_builds_a_model_that_is_not_ready(g):
    """``mlrank`` is set to the largest rank of every mode through the setter, then the model is built."""
    from polara_b200 import pipelines
    c = "b_"
    model = stand_alone_model(g, c)
    a = case_arrays(g, c)
    model.factors = {}
    model._mlrank = (2, 2, 2)
    model._is_ready = False
    built = []

    def build():
        built.append(model.mlrank)
        model.factors = {"userid": a["u0"], "itemid": a["u1"], "rating": a["u2"], "core": a["core"]}
        model._is_ready = True
    model.build = build
    _stub_sweep(g, c, model, [])
    best = pipelines.find_optimal_tucker_ranks(model, tucker_ranks(g, c), "recall", same_space=True, verbose=True,
                                               metric_type="relevance")
    assert built == [tuple(int(x) for x in a["mlrank"])] and best == tuple(int(x) for x in g[c + "best"])
    assert model.verbose is False


def test_sweep_argument_errors(g):
    """refused before any device work: a triple wider than the build, an item-sharded model, a callable or non-linear
    flattener."""
    model = stand_alone_model(g, "a_")
    for bad in ([(11, 8, 4)], [(10, 9, 4)], [(10, 8, 5)], [(0, 8, 4)], [(10, 8)]):
        with pytest.raises(ValueError, match="rebuild"):
            model.tucker_rank_sweep(bad)
    model.flattener = lambda s: s.sum(-1)
    with pytest.raises(NotImplementedError, match="callable"):
        model.tucker_rank_sweep([(10, 8, 4)])
    model.flattener = (slice(None), "max")
    with pytest.raises(NotImplementedError, match="linear"):
        model.tucker_rank_sweep([(10, 8, 4)])
    model.flattener = None
    model.shard = object()
    with pytest.raises(NotImplementedError, match="sharded"):
        model.tucker_rank_sweep([(10, 8, 4)])

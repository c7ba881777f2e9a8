"""Item cold start on the device: the four stand-alone cold-start models against the recorded reference runs
(tests/golden/coldstart_cases.npz) at the built and at a lower rank, their lists bit for bit against the fused scoring
kernel and the exact host emulation, the drop-in on polara's ItemColdStartData without lightfm, the rank search and
repeat runs.  H100 only."""
import sys

import numpy as np
import pytest

from oracle import cholmod_stub
from oracle import coldstart_oracle as co
from oracle import hybrid_oracle as ho
from tests.helpers import check_topk_against_scores, subspace_gap

pytestmark = pytest.mark.gpu

CLASSES = {"SVDModelItemColdStart": "B200SVDModelItemColdStart", "ScaledSVDItemColdStart": "B200ScaledSVDItemColdStart",
           "HybridSVDItemColdStart": "B200HybridSVDItemColdStart",
           "ScaledHybridSVDItemColdStart": "B200ScaledHybridSVDItemColdStart"}


def _cases():
    from tests.conftest import load_golden
    return [str(c) for c in load_golden("coldstart_cases")["cases"]]


def _model(c, rank=None, iters=12):
    """the stand-alone class of the recorded case on its ColdStartData, configured as the reference run was."""
    import polara_b200.models as pm
    model = getattr(pm, CLASSES[str(c["model"])])(co.data(c))
    model.verbose = False
    model.rank = int(c["rank"]) if rank is None else rank
    model.topk = int(c["topk"])
    model.power_iters = iters
    if bool(c["scaled"]):
        model.col_scaling, model.row_scaling = float(c["col_scaling"]), float(c["row_scaling"])
    if bool(c["hybrid"]):
        sim = co.csr(c, "item_sim")
        factor = cholmod_stub.cholesky(sim, beta=ho.beta(float(c["features_weight"])))
        np.testing.assert_array_equal(factor.P(), c["item_perm"])
        model.item_cholesky_factor = (factor.L(), factor.P())
    return model


def _check_lists(model, c, recs, recorded):
    """>= 97 % of the entries equal the reference's, and every list is a valid top-k of the f64 scores of the model's
    own factors, W and transform (tie-aware), with >= 99 % of the entries exact."""
    assert recs.shape == recorded.shape and recs.dtype == np.int64
    assert (recs == recorded).mean() > 0.97
    f = model.data.fields
    u, s = model.factors[f.userid], model.factors["singular_values"]
    w, t = model.item_features_embeddings, model._item_features_transform_helper
    fc = model.data.cold_item_features
    own = co.scores(fc, w, t, u, s)
    e = np.asarray(fc @ w) @ t
    tol = 4e-6 * np.abs(e).sum(1).max() * np.abs(u * s[None, :]).max()
    assert check_topk_against_scores(recs, own, [], [], int(c["topk"]), tol) >= 0.99


def _check_metrics(model, c, recorded):
    """evaluate(): hits within 3 of the reference; precision, recall, MAP, ARHR and coverage equal evaluate_lists on
    the model's own lists (ndcg / ndcl are garbage in the reference and never compared)."""
    from polara_b200.host import evaluate_lists
    rel, rank, exp, hits = model.evaluate()
    assert abs(hits.true_positive - recorded[10]) <= 3 and abs(hits.false_negative - recorded[13]) <= 3
    h = model.data.test.holdout
    want = evaluate_lists(model.recommendations, h["itemid_cold"].values, h["userid"].values, None,
                          int(c["n_users"]))
    assert (rel.precision, rel.recall, rank.map, rank.arhr, exp.coverage) == \
        (want[0].precision, want[0].recall, want[1].map, want[1].arhr, want[2].coverage)


@pytest.mark.parametrize("name", _cases())
def test_model_reproduces_the_reference_runs(golden, name):
    """build, lists and metrics at the built rank; then ``rank = low_rank`` truncates W with the factors and recomputes
    the transform without a rebuild or a re-upload of U diag(s); raising the rank back clears the factors and
    ``recommendations`` rebuilds."""
    c = co.case(golden("coldstart_cases"), name)
    model = _model(c)
    model.build()
    f = model.data.fields
    np.testing.assert_allclose(model.factors["singular_values"], c["singular_values"], rtol=2e-4)
    assert subspace_gap(model.factors[f.itemid], c["item_factors"]) < 2e-2
    assert subspace_gap(model.factors[f.userid], c["user_factors"]) < 2e-2
    w_src = model.factors["itemid_projector_right" if bool(c["hybrid"]) else f.itemid]
    np.testing.assert_allclose(model.item_features_embeddings, co.feature_mapping(model.data.item_features, w_src),
                               rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(model._item_features_transform_helper, co.transform(model.item_features_embeddings),
                               rtol=1e-9)
    recs = model.get_recommendations()
    _check_lists(model, c, recs, c["recs"])
    _check_metrics(model, c, c["evaluate"])
    users_dev = model._dev_scaled_users[2]

    low = int(c["low_rank"])
    model.rank = low
    assert model._is_ready and model.item_features_embeddings.shape[1] == low
    np.testing.assert_allclose(model._item_features_transform_helper, co.transform(model.item_features_embeddings),
                               rtol=1e-9)
    recs_low = model.get_recommendations()
    assert model._dev_scaled_users[2] is users_dev                      # the cached operand served the lower rank
    _check_lists(model, c, recs_low, c["recs_low"])
    _check_metrics(model, c, c["evaluate_low"])

    model.rank = int(c["rank"])
    assert not model._is_ready and model.item_features_embeddings is None
    again = model.recommendations                                         # rebuilds
    assert model._is_ready and model.item_features_embeddings.shape[1] == int(c["rank"])
    np.testing.assert_array_equal(again, recs)


@pytest.mark.parametrize("name", ["svd", "hybrid"])
@pytest.mark.parametrize("rank", [None, "low"])
def test_lists_are_bit_exact_on_the_same_operands(golden, name, rank):
    """the model's lists equal pb200_score_topk (SIMT) on the same fp32 E_cold and U diag(s), and the exact host
    emulation of the canonical chain (ids and order, no tolerance)."""
    from polara_b200.engine import round_up
    from tests.exact_scoring import canonical_scores, expected_lists
    c = co.case(golden("coldstart_cases"), name)
    model = _model(c)
    model.build()
    if rank == "low":
        model.rank = int(c["low_rank"])
    r = model.factors["singular_values"].shape[0]
    recs = model.get_recommendations()
    eng = model.engine
    w = model.item_features_embeddings[:, :r] @ model._item_features_transform_helper
    ld = round_up(r, 32)
    w_pad = np.zeros((w.shape[0], ld), np.float32)
    w_pad[:, :r] = w
    fc = model.data.cold_item_features
    fc.sort_indices()
    f_dev = eng.upload_csr(fc.indptr.astype(np.int64), fc.indices.astype(np.int32), fc.data.astype(np.float32), fc.shape)
    e = eng.spmm(f_dev, eng.upload(w_pad), ell=ld)
    u = model.factors["userid"]
    us = np.zeros((u.shape[0], ld), np.float32)
    us[:, :r] = u * model.factors["singular_values"][None, :r]
    with eng.score_kernel_scope("simt"):
        simt = eng.score_topk(e, eng.upload(us), r, model.topk).cpu().numpy()
    np.testing.assert_array_equal(recs, simt)
    want, _ = expected_lists(canonical_scores(e.cpu().numpy(), us, r), None, model.topk)
    np.testing.assert_array_equal(recs, want)


def test_second_build_and_second_call_give_the_same_bits(golden):
    c = co.case(golden("coldstart_cases"), "scaled_hybrid")
    model = _model(c)
    model.build()
    first = {k: np.array(v) for k, v in model.factors.items()}
    transform = model._item_features_transform_helper.copy()
    recs = model.get_recommendations()
    np.testing.assert_array_equal(model.get_recommendations(), recs)
    model.build()
    for key, val in first.items():
        np.testing.assert_array_equal(model.factors[key], val, err_msg=key)
    np.testing.assert_array_equal(model._item_features_transform_helper, transform)
    np.testing.assert_array_equal(model.get_recommendations(), recs)


def test_find_optimal_svd_rank_runs_the_reference_loop(golden):
    """on a cold-start model the rank search returns what the reference's loop gives on the same model (``rank = r``,
    recommendations, evaluate, ranks descending), and leaves rank, factors and transform as they were."""
    from polara_b200.pipelines import evaluate_models, find_optimal_svd_rank
    c = co.case(golden("coldstart_cases"), "svd")
    model = _model(c)
    model.build()
    ranks = [3, 7, 12]
    full = dict(model.factors)
    transform = model._item_features_transform_helper
    best, scores = find_optimal_svd_rank(model, ranks, "recall", return_scores=True)
    assert model.rank == 12 and model._item_features_transform_helper is transform
    assert all(model.factors[k] is v for k, v in full.items())
    loop = {}
    for rank in sorted(ranks, reverse=True):
        model.rank = rank
        loop[rank] = evaluate_models(model, "recall")[model.method]
        model._recommendations = None
    assert list(scores.index) == ranks and [scores.loc[r] for r in ranks] == [loop[r] for r in ranks]
    assert best == max(loop, key=loop.get)
    assert scores.name == "PureSVD(cs)"


def test_dropin_on_polaras_item_cold_start_data_without_lightfm(golden, monkeypatch):
    """dropin_coldstart() on polara's ItemColdStartData / ItemColdStartSimilarityData, with ``lightfm`` not importable:
    the same split as the recorded runs, so the lists and hits follow the reference's."""
    from oracle import ref_driver as rd
    if rd.reference_root() is None:
        pytest.skip("reference not installed (oracle/_ref)")
    monkeypatch.setitem(sys.modules, "lightfm", None)                    # import lightfm -> ImportError
    rd.import_reference()
    import polara.recommender.hybrid.models as hm
    from oracle import make_coldstart_golden as mk
    from polara_b200.models import dropin_coldstart
    monkeypatch.setattr(hm, "cholesky_decomp_sparse", cholmod_stub.cholesky, raising=False)
    g = golden("coldstart_cases")
    factories = {name: (factory, cfg) for name, _, factory, cfg in mk.datasets()}
    for name, cls in zip(("svd", "scaled_svd", "hybrid", "scaled_hybrid"), dropin_coldstart()):
        c = co.case(g, name)
        factory, cfg = factories[name]
        data = factory()
        model = cls(data)
        model.verbose = False
        if "features_weight" in cfg:
            model._sparse_mode = True
            model.features_weight = cfg["features_weight"]
        model.rank, model.topk = int(c["rank"]), int(c["topk"])
        model.build()
        np.testing.assert_allclose(model.factors["singular_values"], c["singular_values"], rtol=2e-4)
        recs = model.get_recommendations()
        assert recs.shape == c["recs"].shape and (recs == c["recs"]).mean() > 0.97
        hits = model.evaluate("hits")
        assert abs(hits.true_positive - c["evaluate"][10]) <= 3
        assert model.method == ("PureSVD(cs)" if "hybrid" not in name else "HybridSVD(cs)") + \
            ("-s" if name.startswith("scaled") else "")
    assert "polara.recommender.coldstart.models" not in sys.modules

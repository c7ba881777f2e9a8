"""Rank sweeps on the device: pb200_sampled_topk_ranks against pb200_sampled_topk at each rank (bit for bit, both map
paths), the standard sweep against the fused scoring kernel on prefix copies of the same embeddings (bit for bit) and
against f64, and the device find_optimal_svd_rank against the reference's recorded search
(tests/golden/rank_sweep.npz, oracle/make_rank_sweep_golden.py)."""
import os

import numpy as np
import pytest
import scipy.sparse as sps
import torch

from tests.helpers import check_topk_against_scores
from tests.test_gpu_sampler import DEFAULT_SLOTS, _scale_lists, _slots_for
from tests.test_oracle_rank_sweep import stand_alone_model

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rank_sweep.npz")
RANK_SETS = ([1], [1, 2, 3, 5, 8], list(range(10, 151, 10)))
WIDTH = 150                                        # lde = ldv = the largest rank of the last set


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    e = get_engine(0)
    yield e
    e.set_sampler_map_slots(DEFAULT_SLOTS)
    e.set_score_kernel("tc")


def _bits(t):
    return t.cpu().numpy().view(np.uint32)


def _problem(rng, m, n, h, lens):
    """factors of width WIDTH with exact ties (item 7 = item 3, both often held out), random exclusion lists, holdout
    ids that include ids out of range."""
    e = rng.standard_normal((m, WIDTH)).astype(np.float32)
    v = rng.standard_normal((n, WIDTH)).astype(np.float32)
    v[7] = v[3]
    v[11] = v[3]
    indptr = np.zeros(m + 1, np.int64)
    np.cumsum(lens, out=indptr[1:])
    indices = np.concatenate([rng.permutation(n)[:L] for L in lens]).astype(np.int32)
    hold = rng.integers(0, n, (m, h)).astype(np.int64)
    if h:
        hold[::5, 0] = 3
        hold[1::7, -1] = -1
        hold[2::7, 0] = n
    return e, v, indptr, indices, hold


def _check_against_single(eng, e_d, v_d, ranks, hold_d, ip_d, ix_d, seeds, s, k):
    pos, sc = eng.sampled_topk_ranks(e_d, v_d, ranks, hold_d, ip_d, ix_d, seeds, s, k, want_scores=True)
    st = eng.sampler_stats()
    assert pos.shape == (len(ranks), ip_d.shape[0] - 1, k)
    for j, r in enumerate(ranks):
        p1, s1 = eng.sampled_topk(e_d, v_d, r, hold_d, ip_d, ix_d, seeds, s, k, want_scores=True)
        np.testing.assert_array_equal(pos[j].cpu().numpy(), p1.cpu().numpy(), err_msg="rank %d" % r)
        np.testing.assert_array_equal(_bits(sc[j]), _bits(s1), err_msg="rank %d" % r)
    pos2, sc2 = eng.sampled_topk_ranks(e_d, v_d, ranks, hold_d, ip_d, ix_d, seeds, s, k, want_scores=True)
    np.testing.assert_array_equal(pos2.cpu().numpy(), pos.cpu().numpy())
    np.testing.assert_array_equal(_bits(sc2), _bits(sc))
    return pos, st


@pytest.mark.parametrize("path", ["smem", "global"])
@pytest.mark.parametrize("h", [0, 1, 3])
def test_kernel_equals_single_rank_calls(eng, path, h):
    rng = np.random.default_rng(100 + h)
    m, n, s = 700, 2500, 60
    lens = rng.integers(0, 900, m)
    lens[:3] = (0, 1, n - s - h)                        # empty list, one item, exactly s + h items left
    e, v, indptr, indices, hold = _problem(rng, m, n, h, lens)
    e_d, v_d = eng.upload(e), eng.upload(v)
    ip_d, ix_d, hold_d = eng.upload(indptr), eng.upload(indices), eng.upload(hold)
    seeds = np.random.SeedSequence(h).generate_state(m)
    eng.set_sampler_map_slots(DEFAULT_SLOTS if path == "smem" else 0)
    try:
        for k in sorted({1, 10, 40, h + s}):
            for ranks in RANK_SETS:
                pos, st = _check_against_single(eng, e_d, v_d, ranks, hold_d, ip_d, ix_d, seeds, s, k)
                n_smem = int((_slots_for(lens, s) <= DEFAULT_SLOTS).sum()) if path == "smem" else 0
                assert (st["smem_users"], st["global_users"]) == (n_smem, m - n_smem)
                assert st["launches"] == 1 + (n_smem > 0) + (n_smem < m)
                if h and k == h + s:
                    # an out-of-range holdout id is NaN at every rank: never listed, so the row has a -1 pad
                    assert (pos[:, 1, :] == -1).any(dim=1).all() and (pos[:, 2, :] == -1).any(dim=1).all()
                    assert not (pos[:, 1, :] == h - 1).any() and not (pos[:, 2, :] == 0).any()
    finally:
        eng.set_sampler_map_slots(DEFAULT_SLOTS)


def test_kernel_at_c2_like_exclusion_lengths(eng):
    """2e5 users with C2-like exclusion lengths, users at the shared-memory threshold and heavy users."""
    rng = np.random.default_rng(78)
    m, n, s, k = 200_000, 100_000, 999, 10
    indptr, indices, heavy, thr = _scale_lists(rng, m, n, s)
    lens = np.diff(indptr)
    e = (rng.standard_normal((m, WIDTH)) / 4).astype(np.float32)
    v = (rng.standard_normal((n, WIDTH)) / 4).astype(np.float32)
    hold = rng.integers(0, n, (m, 1)).astype(np.int64)
    seeds = np.random.SeedSequence(4).generate_state(m)
    e_d, v_d = eng.upload(e), eng.upload(v)
    _, st = _check_against_single(eng, e_d, v_d, RANK_SETS[2], eng.upload(hold), eng.upload(indptr),
                                  eng.upload(indices), seeds, s, k)
    n_glob = int((_slots_for(lens, s) > DEFAULT_SLOTS).sum())
    assert st["global_users"] == n_glob >= 10 and st["smem_users"] == m - n_glob
    assert st["launches"] == 3


def test_errors(eng):
    rng = np.random.default_rng(9)
    m, n, s = 50, 300, 20
    e, v, indptr, indices, hold = _problem(rng, m, n, 1, rng.integers(0, 200, m))
    args = lambda ix: (eng.upload(hold), eng.upload(indptr), eng.upload(ix),      # noqa: E731
                       np.random.SeedSequence(0).generate_state(m), s, 5)
    e_d, v_d = eng.upload(e), eng.upload(v)
    for ranks, msg in (([], "1..64"), (list(range(1, 66)), "1..64"), ([3, 2], "ascending"), ([2, 2], "ascending"),
                       ([0, 4], ">= 1"), ([4, WIDTH + 1], "exceeds")):
        with pytest.raises(ValueError, match=msg):
            eng.sampled_topk_ranks(e_d, v_d, ranks, *args(indices))
    assert len(eng.sampled_topk_ranks(e_d, v_d, list(range(1, 65)), *args(indices))) == 64
    with pytest.raises(ValueError, match="exceeds"):                          # ldv narrower than lde
        eng.sampled_topk_ranks(e_d, eng.upload(v[:, :40].copy()), [10, 41], *args(indices))
    bad = indices.copy()
    bad[5] = n
    with pytest.raises(ValueError, match="outside"):
        eng.sampled_topk_ranks(e_d, v_d, [4, 8], *args(bad))
    with pytest.raises(ValueError, match="fewer than"):
        eng.sampled_topk_ranks(e_d, v_d, [4, 8], eng.upload(hold), eng.upload(indptr), eng.upload(indices),
                               np.zeros(m, np.uint32), n + 1, 5)
    with pytest.raises(ValueError, match="k must be"):
        eng.sampled_topk_ranks(e_d, v_d, [4, 8], eng.upload(hold), eng.upload(indptr), eng.upload(indices),
                               np.zeros(m, np.uint32), s, s + 2)


# ---------------------------------------------------------------- standard protocol ---------------------------------
def _standard_model(projectors, seed=12):
    from polara_b200.host import ArrayData
    from polara_b200.models import B200SVDModel
    from polara_b200.synth import planted_ratings
    m, n, width = 900, 1300, 48
    u, i, r = planted_ratings(m, n, 30, rank=8, seed=seed)
    a = sps.csr_matrix((r.astype(np.float64), (u, i)), shape=(m, n))
    a.sum_duplicates()
    coo = a.tocoo()
    data = ArrayData(np.stack([coo.row, coo.col], axis=1), coo.data, a.shape, test_user=coo.row, test_item=coo.col,
                     test_fdbk=coo.data, test_shape=a.shape)
    model = B200SVDModel(data)
    model.verbose = False
    model.rank = width
    rng = np.random.default_rng(seed)
    v = np.linalg.qr(rng.standard_normal((n, width)))[0]
    model.factors = {"userid": None, "itemid": v, "singular_values": np.ones(width)}
    if projectors:
        model.factors["itemid_projector_left"] = v * rng.uniform(0.5, 1.5, (n, 1))
        model.factors["itemid_projector_right"] = v * rng.uniform(0.5, 1.5, (n, 1))
    model._is_ready = True
    model.topk = 10
    return model, a


@pytest.mark.parametrize("projectors", [False, True])
@pytest.mark.parametrize("kernel", ["tc", "simt"])
@pytest.mark.parametrize("filter_seen", [True, False])
def test_standard_sweep_equals_prefix_scoring(eng, kernel, filter_seen, projectors):
    from polara_b200.engine import round_up
    model, a = _standard_model(projectors)
    model.score_kernel = kernel
    model.filter_seen = filter_seen
    ranks = [1, 5, 17, 32, 33, 48]
    lists = model.rank_sweep(ranks[::-1])
    assert sorted(lists) == ranks
    # E_max as the sweep forms it, then each rank on zero-padded prefix copies
    test_data, shape, _ = model._get_test_data()
    p_dev, seen = model._test_csr_device(test_data, shape)
    v_fold, v_score = model._item_projector_device(model._device_factor("itemid"))
    e_max = eng.spmm(p_dev, v_fold, ell=min(v_fold.shape[1], round_up(ranks[-1], 32)))
    eng.set_score_kernel(kernel)
    f = model.factors
    vr = f["itemid_projector_right"] if projectors else f["itemid"]
    vl = f["itemid_projector_left"] if projectors else f["itemid"]
    for r in ranks:
        ld = round_up(r, 32)
        e_r = torch.zeros((shape[0], ld), dtype=torch.float32, device=eng.device)
        v_r = torch.zeros((shape[1], ld), dtype=torch.float32, device=eng.device)
        e_r[:, :r] = e_max[:, :r]
        v_r[:, :r] = v_score[:, :r]
        want = eng.score_topk(e_r, v_r, r, model.topk, seen=seen if filter_seen else None).cpu().numpy()
        np.testing.assert_array_equal(lists[r], want, err_msg="rank %d" % r)
        # against f64 at this rank
        e64 = a.dot(vr[:, :r].astype(np.float32).astype(np.float64))
        s64 = e64 @ vl[:, :r].astype(np.float32).astype(np.float64).T
        tol = 4e-6 * np.abs(e64).sum(1).max() * np.abs(vl[:, :r]).max() + 1e-12
        rows, cols = (a.nonzero() if filter_seen else ([], []))
        assert check_topk_against_scores(lists[r], s64, rows, cols, model.topk, tol) >= 0.99, r


# ----------------------------------------------------------------------------- golden --------------------------------
def _near_tie_bound(mine, ref):
    """a per-user mean metric can move by at most 1 / n_users for each row whose list differs"""
    return (mine != ref).any(axis=1).sum() / mine.shape[0] + 1e-12


def test_sampled_sweep_reproduces_the_reference(g, eng):
    model = stand_alone_model(g, "s_")
    ranks = [int(r) for r in g["s_ranks"]]
    hold = g["s_holdout_item"].reshape(-1, 1)
    lists = model.sampled_rank_sweep(ranks, hold, n_unseen=int(g["s_n_unseen"]), seed=int(g["s_data_seed"]),
                                     holdout_users=g["s_holdout_user"])
    for r in ranks:
        assert (lists[r] == g["s_lists_r%d" % r]).mean() >= 0.995, r
    # pre-sampled: the same draw handed over explicitly gives the same lists
    from oracle import sampler_oracle as so
    from polara_b200.models import sampled_exclusion_lists
    test = (g["s_test_user"], g["s_test_item"], g["s_test_fdbk"])
    shape = tuple(int(x) for x in g["s_shape"])
    indptr, indices = sampled_exclusion_lists(test, shape, hold, g["s_holdout_user"])
    drawn = so.sample_rows(indptr, indices, shape[1], int(g["s_n_unseen"]),
                           np.random.SeedSequence(int(g["s_data_seed"])).generate_state(shape[0]))
    pre = model.sampled_rank_sweep(ranks, hold, drawn)
    for r in ranks:
        np.testing.assert_array_equal(pre[r], lists[r])


def _search_like_the_reference(g, model, case):
    """the device find_optimal_svd_rank with the fixture's settings; checks the best rank, the lists (>= 99 % equal to
    the reference's) and that each score differs from the reference's only through the rows whose lists differ.
    Returns the lists the evaluator saw and the scores."""
    from polara_b200 import pipelines
    ranks = [int(r) for r in g[case + "ranks"]]
    seen = {}
    target, kw = ("mrr", dict(metric_type="ranking", simple_rates=True)) if case == "s_" else \
        ("recall", dict(metric_type="relevance"))

    def evaluator(m, target_metric, **k):
        seen[m.rank] = np.array(m.recommendations)
        return pipelines.evaluate_models(m, target_metric, **k)
    v = model.factors["itemid"]
    best, scores = pipelines.find_optimal_svd_rank(model, ranks, target, return_scores=True, evaluator=evaluator, **kw)
    assert best == int(g[case + "best"])
    assert list(scores.index) == ranks and model.factors["itemid"] is v and model.rank == max(ranks)
    for j, r in enumerate(ranks):
        ref = g[case + "lists_r%d" % r]
        assert (seen[r] == ref).mean() >= 0.99, r
        assert abs(scores.loc[r] - g[case + "scores"][j]) <= _near_tie_bound(seen[r], ref), r
    return seen, scores


@pytest.mark.parametrize("case", ["s_", "k_"])
def test_device_rank_search_stand_alone(g, eng, case):
    from polara_b200.host import evaluate_lists
    model = stand_alone_model(g, case)
    ranks = [int(r) for r in g[case + "ranks"]]
    seen, scores = _search_like_the_reference(g, model, case)
    if case == "k_":
        # the lists are a valid top-k of the f64 scores at every rank (seen items filtered)
        tu, ti, tf = g["k_test_user"], g["k_test_item"], g["k_test_fdbk"]
        shape = tuple(int(x) for x in g["k_shape"])
        p = sps.csr_matrix((tf, (tu, ti)), shape=shape)
        for r in ranks:
            v = g["k_item_factors"][:, :r]
            s64 = p.dot(v) @ v.T
            tol = 4e-6 * np.abs(p.dot(v)).sum(1).max() * np.abs(v).max()
            assert check_topk_against_scores(seen[r], s64, tu, ti, model.topk, tol) >= 0.99, r
    else:
        got = evaluate_lists(seen[ranks[0]], g["s_holdout_user"], g["s_holdout_pos"], None, 1, "ranking",
                             simple_rates=True)
        assert got.mrr == pytest.approx(scores.loc[ranks[0]], rel=1e-12)


def _reference_or_skip():
    try:
        from oracle.ref_driver import import_reference
        import_reference()
    except ImportError as exc:
        pytest.skip("reference not available: %s" % exc)


@pytest.mark.parametrize("case", ["s_", "k_"])
def test_device_rank_search_dropin(g, eng, case):
    """the reference's own data models with the device classes grafted on (drop-in classes)."""
    _reference_or_skip()
    import pandas as pd
    from polara.recommender.data import RandomSampleEvaluationMixin, RecommenderData
    from polara_b200.models import dropin, dropin_sampled
    from polara_b200.synth import planted_ratings

    class SampledData(RandomSampleEvaluationMixin, RecommenderData):
        pass

    if case == "s_":                                         # the data models of oracle/make_rank_sweep_golden.py
        u, i, r = planted_ratings(700, 420, 40, rank=6, seed=21)
        data = SampledData(pd.DataFrame({"userid": u, "itemid": i, "rating": r}), "userid", "itemid", "rating", seed=5)
        data.holdout_size = 1
    else:
        u, i, r = planted_ratings(600, 380, 36, rank=6, seed=13)
        data = RecommenderData(pd.DataFrame({"userid": u, "itemid": i, "rating": r}), "userid", "itemid", "rating", seed=3)
    data.warm_start = False
    data.verbose = False
    data.prepare()
    if case == "s_":
        data.unseen_items_num = int(g["s_n_unseen"])
        data.adapt_holdout()
        model = dropin_sampled()(data)
    else:
        model = dropin()[0](data)
    model.verbose = False
    v = g[case + "item_factors"]
    model.rank = v.shape[1]
    model.topk = int(g[case + "topk"])
    model.factors = {"userid": None, "itemid": v, "singular_values": np.ones(v.shape[1])}
    model._is_ready = True
    seen, _ = _search_like_the_reference(g, model, case)
    # the drop-in class's own sweep dispatches like its get_recommendations
    ranks = [int(r) for r in g[case + "ranks"]]
    lists = model.rank_sweep(ranks)
    for r in ranks:
        np.testing.assert_array_equal(lists[r], seen[r])

"""The Tucker-rank sweep on the device: pb200_rotate_factor bit for bit against its fp64 chain emulated in numpy,
pb200_csr_values_from_table bit for bit against a fresh pb200_coo_to_csr of the same weights, the sweep's lists against
the exact scoring emulation (tests/exact_scoring.py) and against the per-triple path, and the device
find_optimal_tucker_ranks against the reference's recorded search (tests/golden/tucker_sweep.npz)."""
import numpy as np
import pytest

from tests.exact_scoring import canonical_scores, expected_lists
from tests.helpers import check_topk_against_scores
from tests.test_oracle_tucker_sweep import (GOLDEN, key, stand_alone_model, switch_positive, tucker_ranks,  # noqa: F401
                                            visited)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    e = get_engine(0)
    yield e
    e.set_score_kernel("tc")


def rotate_emulated(v, rot):
    """acc = 0.0; acc = acc + V[:, k] * R[k, :] for k ascending (fp64 multiply, fp64 add), then fp32"""
    acc = np.zeros((v.shape[0], rot.shape[1]), np.float64)
    for k in range(v.shape[1]):
        acc = acc + v[:, k, None] * rot[None, k, :]
    return acc.astype(np.float32)


def _wide_fp64(rng, shape):
    return rng.standard_normal(shape) * np.exp2(rng.integers(-30, 30, size=shape))


# ---------------------------------------------------------------------------------------------------------------------
#  pb200_rotate_factor
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 7, 32, 60, 64, 130])
def test_rotate_factor_bits(eng, K):
    import torch
    from polara_b200.engine import round_up
    rng = np.random.default_rng(K)
    n = 203                                                           # not a multiple of the 32-row block
    v_wide = _wide_fp64(rng, (n, K + 5))
    v_dev = eng.upload(v_wide)[:, 2:2 + K]                            # row stride K + 5, offset start
    for r in range(1, K + 1):
        rot = _wide_fp64(rng, (K, r))
        got = eng.rotate_factor(v_dev, eng.upload(rot)).cpu().numpy()
        assert got.shape == (n, round_up(r, 32))
        want = rotate_emulated(v_wide[:, 2:2 + K], rot)
        np.testing.assert_array_equal(got[:, :r].view(np.uint32), want.view(np.uint32), err_msg="K=%d r=%d" % (K, r))
        assert not got[:, r:].view(np.uint32).any(), "padding not zero (K=%d r=%d)" % (K, r)
    # into a NaN-filled buffer: every padding column is written
    out = torch.full((n, 64), float("nan"), device=eng.device)
    eng.rotate_factor(v_dev, eng.upload(_wide_fp64(rng, (K, 3))), out=out)
    assert not out[:, 3:].cpu().numpy().view(np.uint32).any()


def test_rotate_factor_rejects_bad_shapes(eng):
    v = eng.upload(np.ones((10, 4)))
    with pytest.raises(ValueError):
        eng.rotate_factor(v, eng.upload(np.ones((5, 2))))
    with pytest.raises(ValueError):
        eng.rotate_factor(eng.upload(np.ones((3, 1025))), eng.upload(np.ones((1025, 2))))
    with pytest.raises(TypeError):
        eng.rotate_factor(v.float(), eng.upload(np.ones((4, 2))))


# ---------------------------------------------------------------------------------------------------------------------
#  pb200_coo_to_csr_runs + pb200_csr_values_from_table
# ---------------------------------------------------------------------------------------------------------------------
def _triplets(rng, n_rows, n_cols, nnz, n_levels, sort):
    user = rng.integers(0, n_rows, nnz)
    user[user == 3] = 4                                               # row 3 stays empty
    item = rng.integers(0, n_cols, nnz)                               # duplicates (user, item) are frequent
    lev = rng.integers(0, n_levels, nnz)
    if sort:                                                          # strictly increasing: the ingest's fast path
        keys = np.unique(user * n_cols + item)
        user, item = keys // n_cols, keys % n_cols
        lev = rng.integers(0, n_levels, len(keys))
    return user.astype(np.int64), item.astype(np.int64), lev.astype(np.int64)


def _tables(rng, n_levels):
    wide = (rng.standard_normal(n_levels) * np.exp2(rng.integers(-20, 20, n_levels))).astype(np.float32)
    yield wide
    cancel = wide.copy()
    if n_levels > 1:
        cancel[1] = -cancel[0]                                        # runs of levels 0 and 1 can sum to zero
    yield cancel
    signed_zero = wide.copy()
    signed_zero[0] = -0.0
    yield signed_zero


@pytest.mark.parametrize("sort", [False, True])
@pytest.mark.parametrize("n_levels", [1, 5])
def test_values_from_table_equal_fresh_ingest(eng, sort, n_levels):
    rng = np.random.default_rng(7 + n_levels + 10 * sort)
    n_rows, n_cols = 40, 9
    user, item, lev = _triplets(rng, n_rows, n_cols, 600, n_levels, sort)
    u_d, i_d, l_d = eng.upload(user), eng.upload(item), eng.upload(lev)
    p, perm, run_ptr = eng.coo_to_csr_runs(u_d, i_d, None, (n_rows, n_cols))
    plain = eng.coo_to_csr(u_d, i_d, None, (n_rows, n_cols))
    np.testing.assert_array_equal(p.indptr.cpu().numpy(), plain.indptr.cpu().numpy())
    np.testing.assert_array_equal(p.indices.cpu().numpy(), plain.indices.cpu().numpy())
    np.testing.assert_array_equal(p.values.cpu().numpy(), plain.values.cpu().numpy())
    assert int(p.indptr[4]) == int(p.indptr[3])                       # the empty row
    if not sort:
        assert p.nnz < len(user)                                      # duplicates were summed
    for table in _tables(rng, n_levels):                              # several tables in turn on the same CSR
        eng.csr_values_from_table(p, perm, run_ptr, l_d, eng.upload(table))
        fresh = eng.coo_to_csr(u_d, i_d, eng.upload(table[lev]), (n_rows, n_cols))
        np.testing.assert_array_equal(p.values.cpu().numpy().view(np.uint32), fresh.values.cpu().numpy().view(np.uint32))
        np.testing.assert_array_equal(p.indices.cpu().numpy(), fresh.indices.cpu().numpy())
    if n_levels > 1 and not sort:
        assert (p.values.cpu().numpy() == 0).any()                    # a cancelling run stays a stored zero


def test_values_from_table_rejects_bad_levels(eng):
    user, item = np.array([0, 0, 1], np.int64), np.array([1, 1, 2], np.int64)
    p, perm, run_ptr = eng.coo_to_csr_runs(eng.upload(user), eng.upload(item), None, (2, 3))
    with pytest.raises(ValueError, match="outside the table"):
        eng.csr_values_from_table(p, perm, run_ptr, eng.upload(np.array([0, 3, 1], np.int64)),
                                  eng.upload(np.ones(3, np.float32)))
    with pytest.raises(ValueError):
        eng.csr_values_from_table(p, perm, run_ptr, eng.upload(np.array([0, 1], np.int64)),
                                  eng.upload(np.ones(3, np.float32)))


# ---------------------------------------------------------------------------------------------------------------------
#  sweep lists
# ---------------------------------------------------------------------------------------------------------------------
def _rounded(model, t):
    """the rotations ``mlrank = t`` applies (None where a mode keeps its width) and the rounded feedback factor"""
    from polara_b200.models import round_tucker_core
    f = model.data.fields
    full = [model.factors[e] for e in (f.userid, f.itemid, f.feedback)]
    core, rot = model.factors["core"], [None] * 3
    for mode in range(3):
        if full[mode].shape[1] > t[mode]:
            rot[mode], core = round_tucker_core(core, mode, t[mode])
    return rot, (full[2] if rot[2] is None else full[2].dot(rot[2]))


SWEEP = [(10, 8, 4), (10, 8, 3), (6, 8, 2), (10, 5, 4), (6, 5, 3), (2, 2, 1), (6, 2, 4)]


@pytest.mark.parametrize("flat", [None, [2, 3]])
@pytest.mark.parametrize("filter_seen", [True, False])
@pytest.mark.parametrize("kernel", ["simt", "tc"])
def test_sweep_lists_bit_exact(g, eng, kernel, filter_seen, flat):
    """every list is the exact emulation of the canonical scores of E = P V_r against V_r, where V_r is the emulated
    rotation (or the plain fp32 factor at full width) and P holds the weights of the triple's table"""
    from polara_b200.engine import round_up
    from polara_b200.models import flatten_weights
    model = stand_alone_model(g, "a_")
    model.flattener = flat
    model.filter_seen = filter_seen
    model.score_kernel = kernel
    lists = model.tucker_rank_sweep(SWEEP)
    assert list(lists) == SWEEP
    f = model.data.fields
    (tu, ti, tf), shape, _ = model._get_test_data()
    u_d, i_d = eng.upload(np.asarray(tu, np.int64)), eng.upload(np.asarray(ti, np.int64))
    v = model.factors[f.itemid]
    for t in SWEEP:
        rot, w = _rounded(model, t)
        vr = v.astype(np.float32) if rot[1] is None else rotate_emulated(v, rot[1])
        v_pad = np.zeros((v.shape[0], round_up(t[1], 32)), np.float32)
        v_pad[:, :t[1]] = vr
        table = (w @ flatten_weights(w, flat)).astype(np.float32)
        p = eng.coo_to_csr(u_d, i_d, eng.upload(table[np.asarray(tf, np.int64)]), shape[:2])
        e = eng.spmm(p, eng.upload(v_pad), ell=round_up(t[1], 32))
        seen = (p.indptr.cpu().numpy(), p.indices.cpu().numpy()) if filter_seen else None
        want, _ = expected_lists(canonical_scores(e.cpu().numpy(), v_pad, t[1]), seen, model.topk)
        np.testing.assert_array_equal(lists[t], want, err_msg=str(t))


@pytest.mark.parametrize("kernel", ["simt", "tc"])
def test_sweep_against_the_per_triple_path(g, eng, kernel):
    """bit-identical where r2 is the item factor's width; below it equal up to near-ties of the f64 scores"""
    import scipy.sparse as sps
    from polara_b200.models import flatten_weights
    model = stand_alone_model(g, "a_")
    model.score_kernel = kernel
    lists = model.tucker_rank_sweep(SWEEP)
    f = model.data.fields
    full, full_rank = dict(model.factors), model._mlrank
    (tu, ti, tf), shape, _ = model._get_test_data()
    width = full[f.itemid].shape[1]
    for t in SWEEP:
        model.mlrank = t
        per_triple = model.get_recommendations()
        model.factors, model._mlrank = dict(full), full_rank
        if t[1] == width:
            np.testing.assert_array_equal(lists[t], per_triple, err_msg=str(t))
            continue
        rot, w = _rounded(model, t)
        vr = full[f.itemid].dot(rot[1])
        c = w @ flatten_weights(w, model.flattener)
        p = sps.csr_matrix((c[np.asarray(tf, np.int64)], (tu, ti)), shape=shape[:2])
        s64 = p.dot(vr) @ vr.T
        tol = 4e-6 * np.abs(p).dot(np.abs(vr)).sum(1).max() * np.abs(vr).max()
        for ids in (lists[t], per_triple):
            assert check_topk_against_scores(ids, s64, tu, ti, model.topk, tol) >= 0.99, t


def test_sweep_errors_and_state(g, eng):
    model = stand_alone_model(g, "a_")
    before = model.get_recommendations()
    with pytest.raises(ValueError, match="rebuild"):
        model.tucker_rank_sweep([(10, 8, 4), (10, 9, 4)])
    model.shard = object()
    with pytest.raises(NotImplementedError, match="sharded"):
        model.tucker_rank_sweep([(10, 8, 4)])
    del model.shard
    from polara_b200 import pipelines
    pipelines.find_optimal_tucker_ranks(model, tucker_ranks(g, "a_"), "recall", metric_type="relevance")
    model._recommendations = None
    np.testing.assert_array_equal(model.get_recommendations(), before)


# ---------------------------------------------------------------------------------------------------------------------
#  the reference's recorded search
# ---------------------------------------------------------------------------------------------------------------------
def _near_tie_bound(mine, ref):
    """recall moves by at most (differing rows) / (holdout rows) when lists differ in some rows"""
    return (mine != ref).any(axis=1).sum() / max(1, mine.shape[0]) + 1e-12


def _search_like_the_reference(g, model, c):
    from polara_b200 import pipelines
    seen = {}

    def evaluator(m, target_metric, **k):
        seen[m._mlrank] = np.array(m.recommendations)
        return pipelines.evaluate_models(m, target_metric, **k)
    best, scores = pipelines.find_optimal_tucker_ranks(model, tucker_ranks(g, c), "recall", return_scores=True,
                                                       same_space=bool(g[c + "same_space"]), evaluator=evaluator,
                                                       metric_type="relevance")
    assert list(seen) == visited(g, c)
    assert best == tuple(int(x) for x in g[c + "best"])
    matched = 0
    for t, want in zip(scores.index, g[c + "scores"]):
        ref = g[c + "lists_" + key(t)]
        assert (seen[t] == ref).mean() >= 0.98, t
        if (seen[t] == ref).all():
            matched += 1
            assert scores.loc[t] == pytest.approx(want, rel=1e-12), t
        else:
            assert abs(scores.loc[t] - want) <= _near_tie_bound(seen[t], ref), t
    assert matched >= 1
    return seen


@pytest.mark.parametrize("c", ["a_", "b_"])
def test_device_tucker_search_stand_alone(g, eng, c):
    model = stand_alone_model(g, c)
    _search_like_the_reference(g, model, c)


def _reference_or_skip():
    try:
        from oracle.ref_driver import import_reference
        import_reference()
    except ImportError as exc:
        pytest.skip("reference not available: %s" % exc)


@pytest.mark.parametrize("c", ["a_", "b_"])
def test_device_tucker_search_dropin(g, eng, c):
    """the reference's own data model (the one oracle/make_tucker_sweep_golden.py built) with the drop-in class"""
    _reference_or_skip()
    import pandas as pd
    from polara.recommender.data import RecommenderData
    from polara_b200.models import dropin
    from polara_b200.synth import planted_ratings
    u, i, r = planted_ratings(360, 220, 30, rank=5, seed=11 if c == "a_" else 12)
    data = RecommenderData(pd.DataFrame({"userid": u, "itemid": i, "rating": r}), "userid", "itemid", "rating", seed=0)
    data.verbose = False
    data.prepare()
    data.to_coo(tensor_mode=True)                            # indexes the feedback levels, as the build does
    model = dropin()[2](data)
    model.verbose = False
    ref = stand_alone_model(g, c)
    model.topk, model.switch_positive, model.flattener = ref.topk, ref.switch_positive, ref.flattener
    model.factors = dict(ref.factors)
    model._mlrank = ref._mlrank
    model._is_ready = True
    (tu, ti, tf), _, _ = model._get_test_data()
    np.testing.assert_array_equal(np.asarray(ti), g[c + "test_item"])
    seen = _search_like_the_reference(g, model, c)
    lists = model.tucker_rank_sweep(visited(g, c))
    for t in visited(g, c):
        np.testing.assert_array_equal(lists[t], seen[t])

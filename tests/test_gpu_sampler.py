"""On-the-fly sampled evaluation on the device (pb200_sample_unseen / pb200_sampled_topk) against the reference's own
draws (tests/golden/sampler_cases.npz, made by oracle/make_sampler_golden.py) and the host restatement of its sampler
(oracle/sampler_oracle.py): the sampled ids must be equal bit for bit, on the shared-memory and on the global-memory map
path; the fused ranking must equal the pre-sampled path (gather_dot + topk_dense) bit for bit."""
import os

import numpy as np
import pytest
import scipy.sparse as sps
import torch

from oracle import sampler_oracle as so
from tests.helpers import check_topk_against_scores

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sampler_cases.npz")
POISON = -7
DEFAULT_SLOTS = 3072


def _slots_for(L, s):                       # map_slots_for in csrc/sampler.cu
    need = 2 * L + s
    return need + need // 2 + 32


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    e = get_engine(0)
    yield e
    e.set_sampler_map_slots(DEFAULT_SLOTS)


def _sample(eng, indptr, indices, seeds, n, s, pad=3):
    out = torch.full((len(indptr) - 1, s + pad), POISON, dtype=torch.int64, device=eng.device)
    eng.sample_unseen(eng.upload(np.asarray(indptr, np.int64)), eng.upload(np.asarray(indices, np.int32)), seeds, n, s,
                      out=out)
    res = out.cpu().numpy()
    assert (res[:, s:] == POISON).all(), "padding inside ld_out was written"
    return res[:, :s]


def _kernels(fn):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if getattr(e, "device_type", None) == DeviceType.CUDA and "sampler_" in e.name]


@pytest.mark.parametrize("path", ["smem", "global"])
def test_fixture_cases_bit_exact(g, eng, path):
    eng.set_sampler_map_slots(DEFAULT_SLOTS if path == "smem" else 0)
    try:
        for j in range(int(g["n_cases"])):
            n, s = int(g["c%d_n" % j]), int(g["c%d_s" % j])
            indptr, indices, seeds = g["c%d_indptr" % j], g["c%d_indices" % j], g["c%d_seeds" % j]
            got = _sample(eng, indptr, indices, seeds, n, s)
            np.testing.assert_array_equal(got, g["c%d_out" % j].astype(np.int64), err_msg="case %d (%s)" % (j, path))
            np.testing.assert_array_equal(_sample(eng, indptr, indices, seeds, n, s), got)      # second run
            st = eng.sampler_stats()
            lens = np.diff(indptr)
            n_smem = int((_slots_for(lens, s) <= DEFAULT_SLOTS).sum()) if path == "smem" else 0
            assert (st["smem_users"], st["global_users"]) == (n_smem, len(lens) - n_smem), (j, st)
            assert st["launches"] == 1 + (n_smem > 0) + (n_smem < len(lens))
    finally:
        eng.set_sampler_map_slots(DEFAULT_SLOTS)


def test_path_kernels_are_the_ones_that_ran(g, eng):
    n, s = int(g["c0_n"]), int(g["c0_s"])
    args = (g["c0_indptr"], g["c0_indices"], g["c0_seeds"], n, s)
    names = _kernels(lambda: _sample(eng, *args))
    assert len(names) == 2 and "sampler_check_kernel" in names[0] and "sampler_smem_kernel" in names[1], names
    eng.set_sampler_map_slots(0)
    try:
        names = _kernels(lambda: _sample(eng, *args))
    finally:
        eng.set_sampler_map_slots(DEFAULT_SLOTS)
    assert len(names) == 2 and "sampler_check_kernel" in names[0] and "sampler_gmem_kernel" in names[1], names


def _scale_lists(rng, m, n, s):
    """C2-like exclusion lengths (heavy-tailed, median ~40) with a few users in the tens of thousands and users right at
    the map-size threshold of the default budget; ids drawn with replacement, in draw order (unsorted)."""
    lens = np.minimum(np.round(rng.lognormal(3.7, 0.9, m)).astype(np.int64) + 1, n - s)
    heavy = np.arange(5) * 7 + 3
    lens[heavy] = [12000, 25000, 38000, 51000, n - s]
    edge = 514                                     # 2 * 514 + 999 = 2027 -> 3072 slots: the largest shared-memory map
    assert _slots_for(edge, s) <= DEFAULT_SLOTS < _slots_for(edge + 1, s)
    thr = np.arange(10) * 11 + 101
    lens[thr[:5]] = edge
    lens[thr[5:]] = edge + 1
    indptr = np.zeros(m + 1, np.int64)
    np.cumsum(lens, out=indptr[1:])
    indices = rng.integers(0, n, int(indptr[-1]), dtype=np.int64).astype(np.int32)
    return indptr, indices, heavy, thr


def test_scale_against_oracle(eng):
    rng = np.random.default_rng(77)
    m, n, s = 200_000, 100_000, 999
    indptr, indices, heavy, thr = _scale_lists(rng, m, n, s)
    seeds = np.random.SeedSequence(3).generate_state(m)
    got = _sample(eng, indptr, indices, seeds, n, s, pad=1)
    st = eng.sampler_stats()
    lens = np.diff(indptr)
    n_glob = int((_slots_for(lens, s) > DEFAULT_SLOTS).sum())
    assert st["global_users"] == n_glob >= 10 and st["smem_users"] == m - n_glob
    check = np.unique(np.concatenate([heavy, thr, np.argsort(lens)[-20:], rng.choice(m, 2000, replace=False)]))
    assert len(check) >= 2000
    want = so.sample_rows(indptr, indices, n, s, seeds, rows=check)
    np.testing.assert_array_equal(got[check], want)


def _factors(rng, m, n, r):
    e = np.zeros((m, 64), np.float32)
    v = np.zeros((n, 64), np.float32)
    e[:, :r] = rng.standard_normal((m, r))
    v[:, :r] = rng.standard_normal((n, r))
    v[7] = v[3]                                              # exact ties between items
    return e, v


@pytest.mark.parametrize("path", ["smem", "global"])
def test_fused_equals_presampled_path(eng, path):
    rng = np.random.default_rng(5)
    m, n, r, h, s, k = 3000, 5000, 50, 1, 999, 10
    e, v = _factors(rng, m, n, r)
    lens = rng.integers(0, 600, m)
    indptr = np.zeros(m + 1, np.int64)
    np.cumsum(lens, out=indptr[1:])
    indices = np.concatenate([rng.permutation(n)[:L] for L in lens]).astype(np.int32)
    hold = np.stack([np.array([indices[indptr[u]]]) if lens[u] else np.array([3]) for u in range(m)]).astype(np.int64)
    seeds = np.random.SeedSequence(11).generate_state(m)
    e_d, v_d = eng.upload(e), eng.upload(v)
    ip_d, ix_d = eng.upload(indptr), eng.upload(indices)
    eng.set_sampler_map_slots(DEFAULT_SLOTS if path == "smem" else 0)
    try:
        items = eng.sample_unseen(ip_d, ix_d, seeds, n, s)
        pos, sc = eng.sampled_topk(e_d, v_d, r, eng.upload(hold), ip_d, ix_d, seeds, s, k, want_scores=True)
        pos2 = eng.sampled_topk(e_d, v_d, r, eng.upload(hold), ip_d, ix_d, seeds, s, k)
    finally:
        eng.set_sampler_map_slots(DEFAULT_SLOTS)
    all_items = torch.cat([eng.upload(hold), items], dim=1)
    users = torch.arange(m, device=eng.device, dtype=torch.int64)[:, None].expand_as(all_items).contiguous()
    scores = eng.gather_dot(e_d, v_d, r, users, all_items)
    ref_pos, ref_sc = eng.topk_dense(scores, k, want_scores=True)
    np.testing.assert_array_equal(pos.cpu().numpy(), ref_pos.cpu().numpy())
    np.testing.assert_array_equal(sc.cpu().numpy().view(np.uint32), ref_sc.cpu().numpy().view(np.uint32))
    np.testing.assert_array_equal(pos2.cpu().numpy(), pos.cpu().numpy())
    # the sampled ids are the reference's draw
    rows = rng.choice(m, 300, replace=False)
    np.testing.assert_array_equal(items.cpu().numpy()[rows], so.sample_rows(indptr, indices, n, s, seeds, rows=rows))


def _run_model(g):
    from polara_b200.host import ArrayData
    from polara_b200.models import B200SVDModel
    shape = tuple(int(x) for x in g["run_shape"])
    data = ArrayData(np.zeros((1, 2), dtype=np.int64), np.ones(1), shape, g["run_test_user"], g["run_test_item"],
                     g["run_test_fdbk"], shape, warm_start=False)
    model = B200SVDModel(data)
    model.verbose = False
    v = g["run_item_factors"]
    model.rank = v.shape[1]
    model.topk = int(g["run_topk"])
    model.factors = {"userid": None, "itemid": v, "singular_values": np.ones(v.shape[1])}
    model._is_ready = True
    return model, shape


def test_against_the_reference_run(g, eng):
    model, shape = _run_model(g)
    hu, hi = g["run_holdout_user"], g["run_holdout_item"]
    tu, ti, tf = g["run_test_user"], g["run_test_item"], g["run_test_fdbk"]
    from polara_b200.models import sampled_exclusion_lists
    indptr, indices = sampled_exclusion_lists((tu, ti, tf), shape, hi.reshape(shape[0], -1), hu)
    np.testing.assert_array_equal(indptr, g["run_excl_indptr"])
    np.testing.assert_array_equal(indices, g["run_excl_indices"])
    n_unseen = int(g["run_n_unseen"])
    seeds = np.random.SeedSequence(int(g["run_data_seed"])).generate_state(shape[0])
    items = eng.sample_unseen(eng.upload(indptr), eng.upload(indices), seeds, shape[1], n_unseen).cpu().numpy()
    np.testing.assert_array_equal(items, g["run_sampled"].astype(np.int64))
    pos = model.sampled_recommendations(hi.reshape(shape[0], -1), None, test_data=(tu, ti, tf), shape=shape,
                                        n_unseen=n_unseen, seed=int(g["run_data_seed"]), holdout_users=hu)
    assert set(model.last_sampled_timings) == {"exclusion_ms", "device_ms"}
    keep = tf != 0
    prof = sps.csr_matrix((tf[keep], (tu[keep], ti[keep])), shape=shape)
    e64 = prof.dot(g["run_item_factors"])
    hold64 = np.einsum("ur,ur->u", e64, g["run_item_factors"][hi])[:, None]
    s64 = np.concatenate([hold64, g["run_unseen_scores"]], axis=1)
    tol = 1e-4 * np.abs(s64).max()
    exact = check_topk_against_scores(pos, s64, [], [], model.topk, tol)
    assert exact >= 0.995, exact
    assert (pos == g["run_positions"]).mean() >= 0.995


def test_errors(g, eng):
    n, s = int(g["c0_n"]), int(g["c0_s"])
    indptr, indices, seeds = g["c0_indptr"], g["c0_indices"], g["c0_seeds"]
    with pytest.raises(ValueError, match="fewer than"):
        _sample(eng, indptr, indices, seeds, n, s + 1)          # case 0 has users with exactly s items left
    bad = indices.copy()
    bad[5] = n
    with pytest.raises(ValueError, match="outside"):
        _sample(eng, indptr, bad, seeds, n, s)
    bad[5] = -1
    with pytest.raises(ValueError, match="outside"):
        _sample(eng, indptr, bad, seeds, n, s)
    model, shape = _run_model(g)
    hi = g["run_holdout_item"].reshape(shape[0], -1)
    test = (g["run_test_user"], g["run_test_item"], g["run_test_fdbk"])
    with pytest.raises(ValueError, match="unspecified"):
        model.sampled_recommendations(hi, None, test_data=test, shape=shape, n_unseen=None, seed=5)
    model.topk = 1 + 4 + 1
    with pytest.raises(ValueError, match="topk"):
        model.sampled_recommendations(hi, None, test_data=test, shape=shape, n_unseen=4, seed=5)
    e = eng.zeros((shape[0], 32))
    v = eng.zeros((shape[1], 32))
    ip, ix = eng.upload(g["run_excl_indptr"]), eng.upload(g["run_excl_indices"])
    with pytest.raises(ValueError, match="k must be"):
        eng.sampled_topk(e, v, 8, eng.upload(hi), ip, ix, g["run_seeds"], 4, 6)


def test_dropin_sampled_draws_like_the_reference(g):
    """the reference's own data model and mixin with the device path grafted on, sampling on the fly."""
    try:
        from oracle.ref_driver import import_reference
        import_reference()
        from polara.recommender.data import RecommenderData, RandomSampleEvaluationMixin
    except ImportError as exc:
        pytest.skip("reference not available: %s" % exc)
    import pandas as pd
    from polara_b200.models import dropin_sampled
    from polara_b200.synth import planted_ratings

    class SampledData(RandomSampleEvaluationMixin, RecommenderData):
        pass

    u, i, r = planted_ratings(700, 420, 40, rank=6, seed=21)        # the data model of the fixture's run
    data = SampledData(pd.DataFrame({"userid": u, "itemid": i, "rating": r}), "userid", "itemid", "rating", seed=5)
    data.holdout_size = 1
    data.warm_start = False
    data.verbose = False
    data.prepare()
    model = dropin_sampled()(data)
    model.verbose = False
    model.rank = 12
    model.topk = 10
    with pytest.raises(ValueError, match="unspecified"):
        model.factors = {"userid": None, "itemid": g["run_item_factors"], "singular_values": np.ones(12)}
        model._is_ready = True
        model.get_recommendations()
    data.unseen_items_num = int(g["run_n_unseen"])
    pos = model.get_recommendations()
    assert pos.shape == g["run_positions"].shape
    assert (pos == g["run_positions"]).mean() >= 0.995

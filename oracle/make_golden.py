"""Generate ``tests/golden/*.npz`` by running the REAL reference (imported from
the checkout named by POLARA_REFERENCE_ROOT).  TEST INFRASTRUCTURE.

    python oracle/make_golden.py

Each fixture stores the hot path's *inputs* exactly as the reference's data
model hands them to the model (``to_coo``, ``_get_test_data``), plus the
reference's *outputs* (factors, recommendations, evaluate() hit counts), so the
fixtures can be replayed where the reference does not exist.
"""
import os
import sys

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.ref_shim import import_reference  # noqa: E402
from polara_b200.synth import planted_ratings  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def _frame(n_users, n_items, per_user, rank, seed):
    u, i, r = planted_ratings(n_users, n_items, per_user, rank=rank, seed=seed)
    return pd.DataFrame({"userid": u, "itemid": i, "rating": r})


def _holdout_arrays(model):
    h = model.data.test.holdout
    f = model.data.fields
    return (h[f.userid].values.astype(np.int64), h[f.itemid].values.astype(np.int64),
            h[f.feedback].values.astype(np.float64))


def _hits(model, **kw):
    hits = model.evaluate("hits", **kw)
    return np.array([-1 if x is None else x for x in hits], dtype=np.float64)


def _relevance(model, **kw):
    rel = model.evaluate("relevance", **kw)
    return np.array([np.nan if x is None else x for x in rel], dtype=np.float64)


def svd_fixture(name, warm_start, rank, scaled=False, feedback_threshold=None, seed=7,
                switch_positive=None):
    polara = import_reference()
    from polara.recommender.data import RecommenderData
    from polara.recommender.models import SVDModel, ScaledSVD
    df = _frame(420, 260, 36, rank=6, seed=seed)
    data = RecommenderData(df, "userid", "itemid", "rating", seed=0)
    data.warm_start = warm_start
    data.verbose = False
    data.prepare()
    model = (ScaledSVD if scaled else SVDModel)(data, feedback_threshold=feedback_threshold)
    model.verbose = False
    model.rank = rank
    model.switch_positive = switch_positive
    model.build()
    recs = model.get_recommendations()
    idx, val, shp = data.to_coo(tensor_mode=False, feedback_threshold=model.feedback_threshold)
    (tu, ti, tf), tshape, tusers = model._get_test_data()
    hu, hi, hf = _holdout_arrays(model)
    out = dict(
        train_idx=idx.astype(np.int64), train_val=val.astype(np.float64), train_shape=np.array(shp),
        test_user=tu.astype(np.int64), test_item=ti.astype(np.int64), test_fdbk=np.asarray(tf, dtype=np.float64),
        test_shape=np.array(tshape), test_users=np.asarray(tusers, dtype=np.int64),
        holdout_user=hu, holdout_item=hi, holdout_fdbk=hf,
        rank=np.array(rank), topk=np.array(model.topk),
        item_factors=model.factors["itemid"], singular_values=model.factors["singular_values"],
        recs=recs.astype(np.int64),
        hits=_hits(model), relevance=_relevance(model),
        warm_start=np.array(warm_start), scaled=np.array(scaled),
        col_scaling=np.array(getattr(model, "col_scaling", 1.0)),
        row_scaling=np.array(getattr(model, "row_scaling", 1.0)),
        feedback_threshold=np.array(np.nan if feedback_threshold is None else feedback_threshold),
        switch_positive=np.array(np.nan if switch_positive is None else switch_positive),
    )
    # reduced-rank replay (models.py:819-832): same factors truncated, no rebuild
    model.rank = rank - 3
    out["recs_reduced"] = model.get_recommendations().astype(np.int64)
    out["rank_reduced"] = np.array(rank - 3)
    # wider list
    model.topk = 25
    out["recs_top25"] = model.get_recommendations().astype(np.int64)
    # unfiltered
    model.filter_seen = False
    model.topk = 10
    out["recs_unfiltered"] = model.get_recommendations().astype(np.int64)
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), **out)
    print(name, "train nnz", len(val), "test users", tshape[0], "hits", out["hits"])


def coffee_fixture(name, mlrank=(6, 5, 3), seed=11, flattener=None):
    polara = import_reference()
    from polara.recommender.data import RecommenderData
    from polara.recommender.models import CoffeeModel
    df = _frame(360, 220, 30, rank=5, seed=seed)
    data = RecommenderData(df, "userid", "itemid", "rating", seed=0)
    data.verbose = False
    data.prepare()
    model = CoffeeModel(data)
    model.verbose = False
    model.mlrank = mlrank
    model.seed = 3
    model.num_iters = 12
    if flattener is not None:
        model.flattener = flattener
    model.build()
    recs = model.get_recommendations()
    idx, val, shp = data.to_coo(tensor_mode=True)
    (tu, ti, tf), tshape, tusers = model._get_test_data()
    hu, hi, hf = _holdout_arrays(model)
    out = dict(
        train_idx=idx.astype(np.int64), train_val=val.astype(np.float64), train_shape=np.array(shp),
        test_user=tu.astype(np.int64), test_item=ti.astype(np.int64), test_fdbk=np.asarray(tf, dtype=np.int64),
        test_shape=np.array(tshape), test_users=np.asarray(tusers, dtype=np.int64),
        holdout_user=hu, holdout_item=hi, holdout_fdbk=hf,
        mlrank=np.array(mlrank), topk=np.array(model.topk), seed=np.array(model.seed),
        num_iters=np.array(model.num_iters), growth_tol=np.array(model.growth_tol),
        u0=model.factors["userid"], u1=model.factors["itemid"], u2=model.factors["rating"],
        core=model.factors["core"], recs=recs.astype(np.int64), hits=_hits(model),
        flattener=np.array(-1 if flattener is None else flattener),
    )
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), **out)
    print(name, "nnz", len(val), "shape", shp, "hits", out["hits"])


def kernel_fixture(name="kernels_small", seed=5):
    """Direct calls of the reference's static kernels on random inputs."""
    polara = import_reference()
    from polara.recommender.models import RecommenderModel
    from polara.preprocessing.matrices import rescale_matrix
    from polara.lib.tensor import ttm3d_seq
    from polara.recommender.utils import get_chunk_size
    from polara.recommender import defaults
    import scipy.sparse as sps
    rng = np.random.default_rng(seed)
    scores = rng.standard_normal((37, 91))
    seen_r = np.repeat(np.arange(37), 6)
    seen_c = np.concatenate([rng.choice(91, 6, replace=False) for _ in range(37)])
    down = scores.copy()
    RecommenderModel.downvote_seen_items(down, (seen_r, seen_c))

    class _K:  # get_topk_elements only needs ``self.topk``
        topk = 7
        topsort = staticmethod(RecommenderModel.topsort)
    top = RecommenderModel.get_topk_elements(_K(), down)
    a = sps.random(60, 45, density=0.15, random_state=3, format="csr")
    a.data = np.rint(1 + 4 * a.data)
    sc_rows = rescale_matrix(a, 0.7, 1)
    sc_cols = rescale_matrix(a, 0.4, 0)
    nnz = 500
    shp = (30, 20, 4)
    idx = np.stack([rng.integers(0, s, nnz) for s in shp], axis=1).astype(np.intp)
    val = rng.random(nnz)
    u = rng.standard_normal((20, 3))
    v = rng.standard_normal((4, 2))
    ttm0 = ttm3d_seq(idx, val, shp, v, u, ((2, 0), (1, 0)))
    old = defaults.memory_hard_limit
    chunks = np.array([get_chunk_size((1_000_000, 100_000), 10, 1),
                       get_chunk_size((6040, 3706), 10, 1)])
    defaults.memory_hard_limit = old
    np.savez_compressed(
        os.path.join(GOLDEN, name + ".npz"), scores=scores, seen_r=seen_r, seen_c=seen_c, downvoted=down,
        topk7=top.astype(np.int64), a_indptr=a.indptr, a_indices=a.indices, a_data=a.data,
        a_shape=np.array(a.shape), sc_rows=sc_rows.toarray(), sc_cols=sc_cols.toarray(),
        ttm_idx=idx.astype(np.int64), ttm_val=val, ttm_shape=np.array(shp), ttm_u=u, ttm_v=v, ttm0=ttm0,
        chunks=chunks)
    print(name, "done")


def live_fixture(name="reference_live"):
    """Reference outputs that tests/test_oracle_vs_reference.py compares the oracle with: the reference's static kernels
    on seeded inputs, HOOI, an SVDModel and a CoffeeModel through RecommenderData.prepare, round_core and the hit-rate /
    reciprocal-rank functions.  The oracle's own inputs are stored with them, so the comparison runs without the reference."""
    import scipy.sparse as sps
    polara = import_reference()
    from polara.recommender.models import RecommenderModel, SVDModel, CoffeeModel
    from polara.recommender.data import RecommenderData
    from polara.preprocessing.matrices import rescale_matrix
    from polara.lib.tensor import hooi
    from polara.recommender.evaluation import assemble_scoring_matrices, get_hr_score, get_rr_scores
    out = {}
    # downvote / topsort / rescale_matrix on random inputs
    for seed in (1, 2):
        rng = np.random.default_rng(seed)
        s = rng.standard_normal((20, 50))
        rows = np.repeat(np.arange(20), 4)
        cols = np.concatenate([rng.choice(50, 4, replace=False) for _ in range(20)])
        ref = s.copy()
        RecommenderModel.downvote_seen_items(ref, (rows, cols))
        out["dv%d_downvoted" % seed] = ref
        out["dv%d_topsort6" % seed] = np.stack([RecommenderModel.topsort(ref[row], 6) for row in range(20)])
        a = sps.random(40, 30, density=0.2, random_state=seed, format="csr")
        for j, (scaling, axis) in enumerate(((0.4, 0), (0.8, 1), (1, 0))):
            out["dv%d_rescaled%d" % (seed, j)] = rescale_matrix(a, scaling, axis).toarray()
    # HOOI
    rng = np.random.default_rng(3)
    shp = (40, 30, 5)
    idx = np.unique(np.stack([rng.integers(0, s, 900) for s in shp], axis=1), axis=0).astype(np.intp)
    ref = hooi(idx, np.ones(len(idx)), shp, (4, 3, 2), num_iters=6, growth_tol=1e-4, seed=5)
    for j in range(3):
        out["hooi_f%d" % j] = ref[j]
    out["hooi_core"] = ref[3]
    # SVDModel through the reference's data model (ML-1M-like density, shrunk to keep the fixture small)
    df = _frame(1200, 740, 166, rank=12, seed=11)
    data = RecommenderData(df, "userid", "itemid", "rating", seed=0)
    data.verbose = False
    data.prepare()
    model = SVDModel(data)
    model.verbose = False
    model.rank = 10
    model.build()
    out["svd_recs"] = model.get_recommendations().astype(np.int32)
    idx, val, shp = data.to_coo(tensor_mode=False)
    out["svd_train_idx"] = idx.astype(np.int32); out["svd_train_val"] = val.astype(np.float32)
    out["svd_train_shape"] = np.array(shp)
    out["svd_sigma"] = model.factors["singular_values"]
    out["svd_v"] = model.factors[data.fields.itemid]
    (tu, ti, tf), tshape, _ = model._get_test_data()
    out["svd_test_u"] = np.asarray(tu, dtype=np.int32); out["svd_test_i"] = np.asarray(ti, dtype=np.int32)
    out["svd_test_f"] = np.asarray(tf, dtype=np.float32); out["svd_test_shape"] = np.array(tshape)
    # CoffeeModel with the reference's default multilinear rank
    df = _frame(1500, 600, 40, rank=6, seed=13)
    data = RecommenderData(df, "userid", "itemid", "rating", seed=0)
    data.verbose = False
    data.prepare()
    model = CoffeeModel(data)
    model.verbose = False
    model.seed = 3
    model.num_iters = 8
    model.build()
    out["cf_recs"] = model.get_recommendations().astype(np.int32)
    idx, val, shp = data.to_coo(tensor_mode=True)
    out["cf_train_idx"] = idx.astype(np.int32); out["cf_train_val"] = val.astype(np.float32)
    out["cf_train_shape"] = np.array(shp)
    out["cf_mlrank"] = np.array(model.mlrank); out["cf_num_iters"] = np.array(model.num_iters)
    out["cf_growth_tol"] = np.array(model.growth_tol); out["cf_seed"] = np.array(model.seed)
    f = data.fields
    for j, key in enumerate((f.userid, f.itemid, f.feedback)):
        out["cf_f%d" % j] = model.factors[key]
    out["cf_core"] = model.factors["core"]
    (tu, ti, tf), tshape, _ = model._get_test_data()
    out["cf_test_u"] = np.asarray(tu, dtype=np.int32); out["cf_test_i"] = np.asarray(ti, dtype=np.int32)
    out["cf_test_f"] = np.asarray(tf, dtype=np.int64); out["cf_test_shape"] = np.array(tshape)
    # round_core
    rng = np.random.default_rng(9)
    core = rng.standard_normal((7, 6, 4))
    out["rc_core"] = core
    for j, (mode, rank) in enumerate(((0, 3), (1, 6), (1, 2), (2, 1), (2, 3))):
        rot, new_core = CoffeeModel.round_core(core, mode, rank)
        out["rc%d_rot" % j] = rot; out["rc%d_core" % j] = new_core
    # hit rate, ARHR, MRR
    for sp in (None, 4):
        rng = np.random.default_rng(12)
        m, n, k = 60, 90, 10
        recs = np.stack([rng.choice(n, k, replace=False) for _ in range(m)])
        hu = np.repeat(np.arange(m), 3)
        hi = np.concatenate([rng.choice(n, 3, replace=False) for _ in range(m)])
        hf = rng.integers(1, 6, size=len(hu)).astype(np.float64)
        holdout = pd.DataFrame({"userid": hu, "itemid": hi, "rating": hf})
        is_positive = None if sp is None else (hf >= sp)
        d = assemble_scoring_matrices(recs, holdout, "userid", "itemid", is_positive, feedback="rating")
        hr, rr = get_hr_score(d[1]), get_rr_scores(d[1])
        out["rates_%s" % sp] = np.array([hr.hr, rr.arhr, rr.mrr], dtype=np.float64)
    np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), **out)
    print(name, "done")


if __name__ == "__main__":
    os.makedirs(GOLDEN, exist_ok=True)
    kernel_fixture()
    svd_fixture("svd_warm_r10", warm_start=True, rank=10)
    svd_fixture("svd_known_r8", warm_start=False, rank=8, switch_positive=4)
    svd_fixture("svd_scaled_r10", warm_start=True, rank=10, scaled=True)
    # NOTE: a feedback_threshold fixture cannot be produced through the full
    # reference stack under pandas>=3 (data.py:790 writes into a read-only
    # ``.values`` view); that semantic (zeroed feedback stays in the seen list,
    # models.py:191-211) is covered through the oracle in tests/test_oracle_golden.py.
    coffee_fixture("coffee_small")
    coffee_fixture("coffee_flat34", flattener=[2, 3], seed=12)
    live_fixture()

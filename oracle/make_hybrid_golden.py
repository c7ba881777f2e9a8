"""Generate ``tests/golden/hybrid_cases.npz`` by running the REAL reference's HybridSVD and ScaledHybridSVD
(polara/recommender/hybrid/models.py:335-397) on seeded ``SimilarityDataModel`` splits.  TEST INFRASTRUCTURE; needs the
reference checkout named by POLARA_REFERENCE_ROOT.

    POLARA_REFERENCE_ROOT=... python oracle/make_hybrid_golden.py

scikit-sparse is not needed: ``oracle.cholmod_stub`` stands in for CHOLMOD as the module's ``cholesky_decomp_sparse``,
and sparse mode is switched on.  Stored per case ``<name>_*``: the arrays the model reads (training COO, user-sorted
test triplets, shapes, holdout), the similarity matrices in the training index order, the configuration
(features_weight, precompute_auxiliary_matrix, scaled, rank, topk), the permutation of the factor the stub produced for
each side (L itself is deterministic given the similarity matrix and beta, and is recomputed by the tests), the reference's singular values, item factors, both item projectors, its lists and
its ``evaluate('hits')`` counts.
"""
import os
import sys

import numpy as np
import pandas as pd
import scipy.sparse as sps

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import cholmod_stub  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402
from polara_b200.synth import planted_ratings  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "hybrid_cases.npz")


def similarity(n, n_features, per_row, seed):
    """cosine similarity of sparse non-negative features: PSD with a unit diagonal, sparse where rows share no
    feature."""
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(n), per_row)
    cols = np.concatenate([rng.choice(n_features, per_row, replace=False) for _ in range(n)])
    f = sps.csr_matrix((rng.random(len(rows)) + 0.5, (rows, cols)), shape=(n, n_features))
    f = sps.diags(1.0 / np.sqrt(np.asarray(f.multiply(f).sum(1)).ravel())) @ f
    s = (f @ f.T).tocsr()
    s.sort_indices()
    return s


def datasets():
    u, i, r = planted_ratings(400, 200, 25, rank=6, seed=11)
    item_sim = similarity(200, 40, 2, 12)
    user_sim = similarity(400, 80, 2, 13)
    yield "items_w05", (u, i, r), dict(item_sim=item_sim, features_weight=0.5)
    yield "items_w09", (u, i, r), dict(item_sim=item_sim, features_weight=0.9)
    yield "both_w05", (u, i, r), dict(item_sim=item_sim, user_sim=user_sim, features_weight=0.5)
    yield "both_w05_pre", (u, i, r), dict(item_sim=item_sim, user_sim=user_sim, features_weight=0.5, precompute=True)
    yield "items_w09_pre", (u, i, r), dict(item_sim=item_sim, features_weight=0.9, precompute=True)
    yield "scaled_both_w09", (u, i, r), dict(item_sim=item_sim, user_sim=user_sim, features_weight=0.9, scaled=True)


def make_data(arrays, cfg):
    from polara.recommender.hybrid.data import SimilarityDataModel
    u, i, r = arrays
    n_users, n_items = int(u.max()) + 1, int(i.max()) + 1
    mats = {"userid": cfg.get("user_sim"), "itemid": cfg.get("item_sim")}
    idx = {"userid": np.arange(n_users) if mats["userid"] is not None else None,
           "itemid": np.arange(n_items) if mats["itemid"] is not None else None}
    data = SimilarityDataModel(pd.DataFrame({"userid": u, "itemid": i, "rating": r}), "userid", "itemid", "rating",
                               seed=7, relations_matrices=mats, relations_indices=idx)
    data.verbose = False
    data.prepare()
    return data


def _factor_arrays(chol):
    if chol is None:
        return None
    return chol._factor.P().astype(np.int64)


def run_case(name, arrays, cfg, res):
    import polara.recommender.hybrid.models as hm
    hm.cholesky_decomp_sparse = cholmod_stub.cholesky
    data = make_data(arrays, cfg)
    model = (hm.ScaledHybridSVD if cfg.get("scaled") else hm.HybridSVD)(data)
    model._sparse_mode = True
    model.verbose = False
    model.rank = 12
    model.topk = 10
    model.features_weight = cfg["features_weight"]
    model.precompute_auxiliary_matrix = bool(cfg.get("precompute", False))
    model.build()
    recs = model.get_recommendations()
    hits = model.evaluate("hits")
    f = data.fields
    p = name + "_"
    for side, entity in (("item", f.itemid), ("user", f.userid)):
        parts = _factor_arrays(model._cholesky[entity])
        rel = data.get_relations_matrix(entity)
        res[p + side + "_present"] = np.array(parts is not None)
        if parts is not None:
            res[p + side + "_perm"] = parts
            rel = sps.csr_matrix(rel)
            res[p + side + "_sim_indptr"], res[p + side + "_sim_indices"], res[p + side + "_sim_data"] = \
                rel.indptr.astype(np.int64), rel.indices.astype(np.int64), rel.data
    idx, val, tshape = data.to_coo(tensor_mode=False)
    test_data, shape, _ = model._get_test_data()
    tu, ti, tf = test_data
    hold = data.test.holdout
    res.update({p + "train_idx": np.asarray(idx, np.int64), p + "train_val": np.asarray(val),
                p + "train_shape": np.array(tshape, np.int64), p + "test_user": np.asarray(tu, np.int64),
                p + "test_item": np.asarray(ti, np.int64), p + "test_fdbk": np.asarray(tf),
                p + "test_shape": np.array(shape, np.int64), p + "holdout_user": hold[f.userid].values.astype(np.int64),
                p + "holdout_item": hold[f.itemid].values.astype(np.int64), p + "holdout_fdbk": hold[f.feedback].values,
                p + "features_weight": np.array(float(cfg["features_weight"])),
                p + "precompute": np.array(bool(cfg.get("precompute", False))),
                p + "scaled": np.array(bool(cfg.get("scaled", False))),
                p + "col_scaling": np.array(float(getattr(model, "col_scaling", 1.0))),
                p + "row_scaling": np.array(float(getattr(model, "row_scaling", 1.0))),
                p + "rank": np.array(model.rank), p + "topk": np.array(model.topk),
                p + "singular_values": model.factors["singular_values"], p + "item_factors": model.factors[f.itemid],
                p + "projector_left": model.factors["%s_projector_left" % f.itemid],
                p + "projector_right": model.factors["%s_projector_right" % f.itemid],
                p + "recs": np.asarray(recs, np.int64),
                p + "hits": np.array([np.nan if h is None else h for h in hits], np.float64)})
    print("%-16s users %4d items %4d  sigma[0] %.4f sigma[-1] %.4f  hits %s" % (
        name, tshape[0], tshape[1], model.factors["singular_values"][0], model.factors["singular_values"][-1],
        list(res[p + "hits"])))


def main():
    import_reference()
    res = {}
    names = []
    for name, arrays, cfg in datasets():
        run_case(name, arrays, cfg, res)
        names.append(name)
    res["cases"] = np.array(names)
    np.savez_compressed(OUT, **res)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

"""Generate ``tests/golden/coldstart_cases.npz`` by running the REAL reference's item cold-start models
(polara/recommender/coldstart/models.py:225-257: SVDModelItemColdStart, ScaledSVDItemColdStart, HybridSVDItemColdStart,
ScaledHybridSVDItemColdStart) on seeded ``ItemColdStartData`` splits.  TEST INFRASTRUCTURE; needs the reference checkout
named by POLARA_REFERENCE_ROOT.

    POLARA_REFERENCE_ROOT=... python oracle/make_coldstart_golden.py

``polara.recommender.coldstart.models`` imports LightFMWrapper, which imports ``lightfm`` (not needed by the SVD family):
a stub module stands in for it in ``sys.modules`` before the import.  HybridSVD runs on ``oracle.cholmod_stub`` as in
``make_hybrid_golden.py``.  The item features are list-valued genres (1-3 of 20 labels per item); one cold item is
given a label no other item has, so the data model drops it (coldstart/data.py:162-185).  Stored per case ``<name>_*``:
the training COO, the sorted cold holdout (cold id, user, feedback), the user count, the representative users (if any),
the one-hot F of the training items and F_cold of the kept cold items with their shared labels, the factors (U, sigma,
V, the HybridSVD projectors), W and its transform at the built rank, the lists and ``evaluate()`` tuples at the built
rank and at ``low_rank`` (with the transform recomputed there), and for HybridSVD the item similarity matrix and the
stub's permutation.
"""
import os
import sys
import types

import numpy as np
import pandas as pd
import scipy.sparse as sps

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import cholmod_stub  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402
from polara_b200.synth import planted_ratings  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "coldstart_cases.npz")
N_LABELS = 20
RANK, LOW_RANK, TOPK = 12, 7, 10


def stub_lightfm():
    """an importable ``lightfm`` with the one name lightfmwrapper.py:3 reads; the SVD family never calls it."""
    if "lightfm" not in sys.modules:
        mod = types.ModuleType("lightfm")
        mod.LightFM = object
        sys.modules["lightfm"] = mod


def genres(n_items, seed, solo=()):
    """list-valued features: 1-3 distinct labels of N_LABELS per item; the items in ``solo`` get one label of their own."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n_items):
        if i in solo:
            out.append(["solo%d" % i])
        else:
            out.append(["g%02d" % g for g in rng.choice(N_LABELS, rng.integers(1, 4), replace=False)])
    return pd.DataFrame({"genres": out}, index=pd.Index(np.arange(n_items), name="itemid"))


def feature_similarity(features):
    """common-label cosine similarity of the items (PSD, unit diagonal), indexed by the original item id."""
    labels = sorted({g for row in features["genres"] for g in row})
    col = {g: j for j, g in enumerate(labels)}
    rows = np.repeat(np.arange(len(features)), [len(x) for x in features["genres"]])
    cols = [col[g] for x in features["genres"] for g in x]
    f = sps.csr_matrix((np.ones(len(cols)), (rows, cols)), shape=(len(features), len(labels)))
    f = sps.diags(1.0 / np.sqrt(np.asarray(f.sum(1)).ravel())) @ f
    s = (f @ f.T).tocsr()
    s.sort_indices()
    return s


def make_data(frame, features, hybrid, test_sample=None, seed=3):
    from polara.recommender.coldstart.data import ItemColdStartData, ItemColdStartSimilarityData
    if hybrid:
        sim = feature_similarity(features)
        data = ItemColdStartSimilarityData(frame, "userid", "itemid", "rating", seed=seed, item_features=features,
                                           relations_matrices={"userid": None, "itemid": sim},
                                           relations_indices={"userid": None, "itemid": features.index.values})
    else:
        data = ItemColdStartData(frame, "userid", "itemid", "rating", seed=seed, item_features=features)
    data.verbose = False
    data.test_sample = test_sample
    data.prepare()
    return data


def datasets():
    """(name, class name, data factory, extra config).  The first split is made once without a solo item to learn which
    items go cold; the split depends on the seed and the item ids only, so the second construction has the same cold
    set, and its first cold item carries a label no training item has.  Needs the reference on ``sys.path``."""
    u, i, r = planted_ratings(300, 120, 20, rank=6, seed=31)
    frame = pd.DataFrame({"userid": u, "itemid": i, "rating": r})
    probe = make_data(frame, genres(120, 32), False)
    solo = (int(probe.index.itemid.cold_start.old.values[0]),)
    feats = genres(120, 32, solo)
    yield "svd", "SVDModelItemColdStart", lambda: make_data(frame, feats, False), {}
    yield "scaled_svd", "ScaledSVDItemColdStart", lambda: make_data(frame, feats, False, test_sample=0.5), {}
    yield "hybrid", "HybridSVDItemColdStart", lambda: make_data(frame, feats, True), dict(features_weight=0.7)
    yield "scaled_hybrid", "ScaledHybridSVDItemColdStart", lambda: make_data(frame, feats, True, test_sample=0.5), \
        dict(features_weight=0.5)


def _csr(res, key, m):
    m = sps.csr_matrix(m, dtype=np.float64)
    m.sort_indices()
    res[key + "_indptr"], res[key + "_indices"], res[key + "_data"] = \
        m.indptr.astype(np.int64), m.indices.astype(np.int64), m.data
    res[key + "_shape"] = np.array(m.shape, np.int64)


def _evaluate(model):
    out = []
    for t in model.evaluate():
        out.extend(np.nan if x is None else float(x) for x in t)
    return np.array(out, np.float64)


def run_case(name, cls_name, factory, cfg, res):
    import polara.recommender.hybrid.models as hm
    from polara.lib.similarity import stack_features
    stub_lightfm()
    import polara.recommender.coldstart.models as cm
    hm.cholesky_decomp_sparse = cholmod_stub.cholesky
    data = factory()
    model = getattr(cm, cls_name)(data)
    model.verbose = False
    if "features_weight" in cfg:
        model._sparse_mode = True
        model.features_weight = cfg["features_weight"]
    model.rank = RANK
    model.topk = TOPK
    model.build()
    f = data.fields
    cold_col = f.itemid + "_cold"
    p = name + "_"
    labels = model.item_features_labels["genres"]
    res[p + "labels"] = np.array(sorted(labels, key=labels.get))
    _csr(res, p + "F", model.encode_item_features())
    cold_meta = model.item_features.reindex(data.index.itemid.cold_start.old.values, fill_value=[])
    f_cold, _ = stack_features(cold_meta, labels=model.item_features_labels, normalize=False)
    _csr(res, p + "F_cold", f_cold)
    recs = model.get_recommendations()
    ev = _evaluate(model)
    hold = data.test.holdout
    idx, val, tshape = data.to_coo(tensor_mode=False)
    repr_users = data.representative_users
    res.update({p + "model": np.array(cls_name), p + "train_idx": np.asarray(idx, np.int64),
                p + "train_val": np.asarray(val, np.float64), p + "train_shape": np.array(tshape, np.int64),
                p + "n_users": np.array(data.index.userid.training.shape[0]),
                p + "cold_old": data.index.itemid.cold_start.old.values.astype(np.int64),
                p + "cold_new": data.index.itemid.cold_start.new.values.astype(np.int64),
                p + "holdout_cold": hold[cold_col].values.astype(np.int64),
                p + "holdout_user": hold[f.userid].values.astype(np.int64),
                p + "holdout_fdbk": hold[f.feedback].values.astype(np.float64),
                p + "repr_users": (np.zeros(0, np.int64) if repr_users is None
                                   else repr_users.new.values.astype(np.int64)),
                p + "rank": np.array(RANK), p + "low_rank": np.array(LOW_RANK), p + "topk": np.array(TOPK),
                p + "scaled": np.array(cls_name.startswith("Scaled")),
                p + "col_scaling": np.array(float(getattr(model, "col_scaling", 1.0))),
                p + "row_scaling": np.array(float(getattr(model, "row_scaling", 1.0))),
                p + "user_factors": model.factors[f.userid], p + "singular_values": model.factors["singular_values"],
                p + "item_factors": model.factors[f.itemid],
                p + "W": model.item_features_embeddings, p + "transform": model._item_features_transform_helper,
                p + "recs": np.asarray(recs, np.int64), p + "evaluate": ev})
    hybrid = "features_weight" in cfg
    res[p + "hybrid"] = np.array(hybrid)
    if hybrid:
        res[p + "features_weight"] = np.array(float(cfg["features_weight"]))
        res[p + "projector_left"] = model.factors["%s_projector_left" % f.itemid]
        res[p + "projector_right"] = model.factors["%s_projector_right" % f.itemid]
        res[p + "item_perm"] = model._cholesky[f.itemid]._factor.P().astype(np.int64)
        _csr(res, p + "item_sim", data.get_relations_matrix(f.itemid))
    model.rank = LOW_RANK
    res[p + "transform_low"] = model._item_features_transform_helper
    res[p + "recs_low"] = np.asarray(model.get_recommendations(), np.int64)
    model._recommendations = None
    res[p + "evaluate_low"] = _evaluate(model)
    print("%-14s users %d items %d cold %d (of %d in the split) features %d  sigma[0] %.4f  evaluate %s" % (
        name, tshape[0], tshape[1], len(res[p + "cold_new"]), len(np.unique(res[p + "holdout_cold"])),
        len(labels), model.factors["singular_values"][0], np.round(ev, 4).tolist()))


def main():
    import_reference()
    res = {}
    names = []
    for name, cls_name, factory, cfg in datasets():
        run_case(name, cls_name, factory, cfg, res)
        names.append(name)
    res["cases"] = np.array(names)
    np.savez_compressed(OUT, **res)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

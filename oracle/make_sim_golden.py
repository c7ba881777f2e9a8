"""Generate ``tests/golden/sim_cases.npz`` by running the REAL reference's SimilarityAggregation (polara/recommender/
hybrid/models.py:25-44) on a SimilarityDataModel with small generated item relations, and ``tests/golden/
i2i_wide_cases.npz`` from its CooccurrenceModel on a wide, sparse catalogue.  TEST INFRASTRUCTURE; needs the reference
checkout named by POLARA_REFERENCE_ROOT.

    POLARA_REFERENCE_ROOT=... python oracle/make_sim_golden.py

Stored per SIM case ``<name>_*``: the test triplets and shape, the holdout, the data model's ``item_relations`` (CSR
arrays in the training item index, diagonal 1 as SimilarityDataModel sets it), the configuration, the reference's lists
and the form of each chunk's score block (``modes``).  The wide case follows oracle/make_i2i_golden.py's layout.
"""
import os
import sys

import numpy as np
import pandas as pd
import scipy as sp
import scipy.sparse  # noqa: F401

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.make_i2i_golden import long_tail, run_case  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402
from polara_b200.synth import planted_ratings  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "sim_cases.npz")
OUT_WIDE = os.path.join(ROOT, "tests", "golden", "i2i_wide_cases.npz")


def relations(n_items, density, seed, symmetric=True, values="int"):
    """random item x item relations over the original item ids 0..n_items-1."""
    rng = np.random.default_rng(seed)
    nnz = int(density * n_items * n_items)
    r, c = rng.integers(0, n_items, nnz), rng.integers(0, n_items, nnz)
    if values == "int":
        v = rng.integers(1, 6, nnz).astype(np.float64)
    elif values == "dyadic":
        v = rng.integers(-8, 17, nnz) / 8.0                   # exact in binary, some negative, some zero
    else:
        v = rng.random(nnz)
    s = sp.sparse.coo_matrix((v, (r, c)), shape=(n_items, n_items)).tocsr()
    s.sum_duplicates()
    if symmetric:
        s = (s + s.T).tocsr()
    return s


def datasets():
    u, i, r = planted_ratings(600, 300, 20, rank=6, seed=11)
    ratings = (u, i, r.astype(np.int64))
    lt = long_tail(700, 2000, 5, 12)
    yield "sym_dense", ratings, relations(300, 0.05, 1), {}
    yield "sym_sparse", lt, relations(2000, 0.0008, 2), {}
    yield "nonsym", ratings, relations(300, 0.01, 3, symmetric=False), {}
    yield "nonsym_implicit", ratings, relations(300, 0.01, 4, symmetric=False), dict(implicit=True)
    yield "implicit_sparse", lt, relations(2000, 0.0008, 5, symmetric=False), dict(implicit=True, topk=30)
    yield "nofilter", ratings, relations(300, 0.01, 6, symmetric=False), dict(filter_seen=False)
    yield "dyadic", ratings, relations(300, 0.02, 7, symmetric=False, values="dyadic"), {}
    yield "dense_output", ratings, relations(300, 0.01, 8, symmetric=False), dict(dense_output=True)
    yield "float", ratings, relations(300, 0.02, 9, symmetric=False, values="float"), {}


def run_sim_case(name, arrays, rel, cfg, res):
    from polara.recommender import defaults
    from polara.recommender.hybrid.data import SimilarityDataModel
    from polara.recommender.hybrid.models import SimilarityAggregation
    u, i, r = arrays
    n = rel.shape[0]
    data = SimilarityDataModel(pd.DataFrame({"userid": u, "itemid": i, "rating": r}), "userid", "itemid", "rating",
                               seed=7, relations_matrices={"itemid": rel}, relations_indices={"itemid": np.arange(n)})
    data.verbose = False
    data.prepare()
    limit = cfg.get("memory_hard_limit", 1)
    old_limit = defaults.memory_hard_limit
    defaults.memory_hard_limit = limit
    try:
        model = SimilarityAggregation(data)
        model.verbose = False
        model.topk = cfg.get("topk", 10)
        model.filter_seen = cfg.get("filter_seen", True)
        model.implicit = cfg.get("implicit", False)
        model.dense_output = cfg.get("dense_output", False)
        model.build()
        recs = model.get_recommendations()
        test_data, shape, _ = model._get_test_data()
        modes = []
        bounds = model._get_slices_idx(shape)
        for a, b in zip(bounds[:-1], bounds[1:]):
            scores, _ = model.slice_recommendations(test_data, shape, a, b)
            modes.append((a, b, int(not sp.sparse.issparse(scores))))
    finally:
        defaults.memory_hard_limit = old_limit
    rel_t = sp.sparse.csr_matrix(data.item_relations)
    assert data.item_relations.format == "csr"
    hold = data.test.holdout
    f = data.fields
    tu, ti, tf = test_data
    p = name + "_"
    res.update({p + "rel_indptr": rel_t.indptr.astype(np.int64), p + "rel_indices": rel_t.indices.astype(np.int64),
                p + "rel_data": rel_t.data.astype(np.float64), p + "rel_shape": np.array(rel_t.shape, np.int64),
                p + "test_user": np.asarray(tu, np.int64), p + "test_item": np.asarray(ti, np.int64),
                p + "test_fdbk": np.asarray(tf), p + "test_shape": np.array(shape, np.int64),
                p + "holdout_user": hold[f.userid].values.astype(np.int64),
                p + "holdout_item": hold[f.itemid].values.astype(np.int64), p + "holdout_fdbk": hold[f.feedback].values,
                p + "topk": np.array(model.topk), p + "filter_seen": np.array(model.filter_seen),
                p + "implicit": np.array(model.implicit), p + "dense_output": np.array(model.dense_output),
                p + "memory_hard_limit": np.array(float(limit)), p + "recs": np.asarray(recs, np.int64),
                p + "modes": np.array(modes, np.int64)})
    print("%-16s users %4d items %4d  rel nnz %6d  chunks %s  pads %d" % (
        name, shape[0], shape[1], rel_t.nnz, "".join("D" if d else "s" for _, _, d in modes), int((recs < 0).sum())))


def main():
    import_reference()
    res, names = {}, []
    for name, arrays, rel, cfg in datasets():
        run_sim_case(name, arrays, rel, cfg, res)
        names.append(name)
    res["cases"] = np.array(names)
    np.savez_compressed(OUT, **res)
    print(OUT, os.path.getsize(OUT), "bytes")
    # a wide, sparse catalogue for the item-to-item model: most item pairs never co-occur
    wide = {}
    run_case("wide", long_tail(400, 60000, 150, 21, zipf=0.3), {}, wide)
    wide["cases"] = np.array(["wide"])
    np.savez_compressed(OUT_WIDE, **wide)
    print(OUT_WIDE, os.path.getsize(OUT_WIDE), "bytes")


if __name__ == "__main__":
    main()

"""Generate ``tests/golden/i2i_cases.npz`` by running the REAL reference's item-to-item model (CooccurrenceModel,
polara/recommender/models.py:693-725) on seeded RecommenderData splits.  TEST INFRASTRUCTURE; needs the reference
checkout named by POLARA_REFERENCE_ROOT.

    POLARA_REFERENCE_ROOT=... python oracle/make_i2i_golden.py

Stored per case ``<name>_*``: the arrays the model reads (training COO, user-sorted test triplets, shapes, holdout),
the configuration (topk, filter_seen, implicit, dense_output, memory_hard_limit), the reference's lists, the form of each
chunk's score block (``modes`` rows: start, stop, dense -- from ``slice_recommendations`` per slice and
``sp.sparse.issparse``) and the reference's ``evaluate()`` metrics (``metric_names`` / ``metrics``).
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

from oracle.ref_shim import import_reference  # noqa: E402
from polara_b200.synth import planted_ratings  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "i2i_cases.npz")


def long_tail(n_users, n_items, per_user, seed, zipf=0.8):
    """few ratings per user over a catalogue with a Zipf popularity: most users get fewer than topk scored items."""
    rng = np.random.default_rng(seed)
    pop = 1.0 / np.arange(1, n_items + 1) ** zipf
    pop /= pop.sum()
    user, item = [], []
    for u in range(n_users):
        items = rng.choice(n_items, per_user, replace=False, p=pop)
        user.append(np.full(per_user, u))
        item.append(np.sort(items))
    user, item = np.concatenate(user), np.concatenate(item)
    return user, item, rng.integers(1, 6, len(user)).astype(np.int64)


def mixed(seed):
    """heavy users first (their chunks go dense), then users of a few items from a flat catalogue (their chunks stay
    sparse), and a few heavy users again at the end."""
    u1, i1, r1 = planted_ratings(300, 400, 60, rank=6, seed=seed)
    u2, i2, r2 = long_tail(700, 2000, 6, seed + 1, zipf=0.0)
    u3, i3, r3 = planted_ratings(100, 400, 60, rank=6, seed=seed + 2)
    return np.r_[u1, u2 + 300, u3 + 1000], np.r_[i1, i2 + 400, i3], np.r_[r1, r2, r3].astype(np.int64)


def datasets():
    u, i, r = planted_ratings(800, 300, 25, rank=6, seed=1)
    yield "dense", (u, i, r.astype(np.int64)), {}
    lt = long_tail(800, 3000, 5, 2)
    yield "sparse", lt, dict(crafted=True)
    yield "mixed", mixed(3), dict(memory_hard_limit=0.00036)
    yield "implicit", lt, dict(implicit=True)
    yield "implicit_dense", (u, i, r.astype(np.int64)), dict(implicit=True)
    yield "nofilter", lt, dict(filter_seen=False)
    yield "dense_output", lt, dict(dense_output=True)
    # +-1 feedback: item pairs rated both ways by different users cancel to exactly 0 in S and in P S
    us, is_, rs = planted_ratings(900, 120, 6, rank=4, seed=4)
    yield "signed", (us, is_, np.where(rs >= 3, 1, -1).astype(np.int64)), {}
    # non-negative, non-integer values that are exact in float32 (the device ingests float32)
    uf, itf, rf = long_tail(800, 1500, 8, 5)
    vf = np.float32(np.random.default_rng(6).random(len(uf)) * 4 + 0.05).astype(np.float64)
    yield "float", (uf, itf, vf), {}


def _flat_metrics(metrics):
    names, values = [], []
    for group in metrics:
        for field, value in zip(group._fields, group):
            if value is not None:
                names.append("%s.%s" % (type(group).__name__, field))
                values.append(float(value))
    return names, values


def _crafted_lists(recs, data):
    """the reference's lists edited so that a -1 pad of user v + 1 would collide with the largest holdout item H of
    user v under a key ``user * (H + 1) + item``: ids above H and H itself leave user v's list, and v + 1 ends in a pad."""
    hold = data.test.holdout
    f = data.fields
    h_user = np.unique(hold[f.userid].values, return_inverse=True)[1]
    h_item = hold[f.itemid].values
    big = int(h_item.max())
    v = int(h_user[np.flatnonzero(h_item == big)].min())
    if v + 1 >= recs.shape[0]:
        v = recs.shape[0] - 2
        big = int(h_item[h_user == v].max())
    out = np.where(recs > big, -1, recs).astype(np.int64)
    out[v][out[v] == big] = -1
    out[v + 1, -1] = -1
    return out


def run_case(name, arrays, cfg, res):
    from polara.recommender import defaults
    from polara.recommender.data import RecommenderData
    from polara.recommender.models import CooccurrenceModel
    u, i, r = arrays
    data = RecommenderData(pd.DataFrame({"userid": u, "itemid": i, "rating": r}), "userid", "itemid", "rating", seed=7)
    data.verbose = False
    data.prepare()
    limit = cfg.get("memory_hard_limit", 1)
    old_limit = defaults.memory_hard_limit
    defaults.memory_hard_limit = limit
    try:
        model = CooccurrenceModel(data)
        model.verbose = False
        model.topk = 10
        model.filter_seen = cfg.get("filter_seen", True)
        model.implicit = cfg.get("implicit", False)
        model.dense_output = cfg.get("dense_output", False)
        model.build()
        recs = model.get_recommendations()
        test_data, shape, _ = model._get_test_data()
        modes = []
        for a, b in zip(*(lambda s: (s[:-1], s[1:]))(model._get_slices_idx(shape))):
            scores, _ = model.slice_recommendations(test_data, shape, a, b)
            modes.append((a, b, int(not sp.sparse.issparse(scores))))
        metrics = model.evaluate()
        if cfg.get("crafted"):
            crafted = _crafted_lists(recs, data)
            model._recommendations = crafted
            res[name + "_crafted_recs"] = crafted
            res[name + "_crafted_metrics"] = _flat_metrics(model.evaluate())[1]
    finally:
        defaults.memory_hard_limit = old_limit
    names, values = _flat_metrics(metrics)
    idx, val, tshape = data.to_coo(tensor_mode=False)
    hold = data.test.holdout
    f = data.fields
    tu, ti, tf = test_data
    p = name + "_"
    res.update({p + "train_idx": np.asarray(idx, np.int64), p + "train_val": np.asarray(val),
                p + "train_shape": np.array(tshape, np.int64), p + "test_user": np.asarray(tu, np.int64),
                p + "test_item": np.asarray(ti, np.int64), p + "test_fdbk": np.asarray(tf),
                p + "test_shape": np.array(shape, np.int64), p + "holdout_user": hold[f.userid].values.astype(np.int64),
                p + "holdout_item": hold[f.itemid].values.astype(np.int64), p + "holdout_fdbk": hold[f.feedback].values,
                p + "n_items_total": np.array(data.index.itemid.shape[0]), p + "topk": np.array(model.topk),
                p + "filter_seen": np.array(model.filter_seen), p + "implicit": np.array(model.implicit),
                p + "dense_output": np.array(model.dense_output), p + "memory_hard_limit": np.array(float(limit)),
                p + "recs": np.asarray(recs, np.int64), p + "modes": np.array(modes, np.int64),
                p + "metric_names": np.array(names), p + "metrics": np.array(values)})
    print("%-15s users %4d items %4d  chunks %s  pads %d  scores dtype %s" % (
        name, shape[0], shape[1], "".join("D" if d else "s" for _, _, d in modes), int((recs < 0).sum()),
        np.asarray(val).dtype))


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

"""Generate ``tests/golden/tucker_sweep.npz`` by running the REAL reference's Tucker-rank search
(``polara.evaluation.pipelines.find_optimal_tucker_ranks``, pipelines.py:119-160).  TEST INFRASTRUCTURE; needs the
reference checkout named by POLARA_REFERENCE_ROOT.

    POLARA_REFERENCE_ROOT=... python oracle/make_tucker_sweep_golden.py

The search is given an ``evaluator`` that wraps the reference's ``evaluate_models`` (pipelines.py:63-78) and records, at
each triple, ``model.recommendations`` and the rounded item and feedback factors the model shows (``mlrank = t``,
models.py:949-980), so the fixture holds the lists the metrics were computed from.  The data are a planted rating
tensor (``planted_ratings``, ratings 1..5 = 5 feedback levels) split by ``RecommenderData``.  Two cases, one CoffeeModel
build each at the largest rank of every mode, target ``recall`` with ``metric_type='relevance'``:

* ``a_`` -- ranks ([10, 6, 2], [8, 5, 2], [4, 3, 1]): the skip rule ``r1*r2 < r3 or r1*r3 < r2 or r2*r3 < r1`` drops
  triples such as (10, 2, 1) and (2, 8, 1);
* ``b_`` -- ranks ([8, 5, 3], [8, 5, 3], [4, 2]) with ``same_space=True``: only ``r2 == r1``; flattener [2, 3].

Stored per case: the inputs the model reads (training and test triplets, holdout), the reference's factors and core
after the search (the full build, which the search restores), the visited triples in order, each triple's lists
(``<case>lists_<r1>_<r2>_<r3>``) and rounded item / feedback factors, the score Series and the best triple.
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

OUT = os.path.join(ROOT, "tests", "golden", "tucker_sweep.npz")


def _key(t):
    return "%d_%d_%d" % tuple(t)


def case(res, prefix, seed, mlranks, same_space, flattener=None):
    from polara.evaluation.pipelines import evaluate_models, find_optimal_tucker_ranks
    from polara.recommender.data import RecommenderData
    from polara.recommender.models import CoffeeModel
    u, i, r = planted_ratings(360, 220, 30, rank=5, seed=seed)
    data = RecommenderData(pd.DataFrame({"userid": u, "itemid": i, "rating": r}), "userid", "itemid", "rating", seed=0)
    data.verbose = False
    data.prepare()
    model = CoffeeModel(data)
    model.verbose = False
    model.seed = 3
    model.num_iters = 12
    if flattener is not None:
        model.flattener = flattener
    f = data.fields
    visited = []

    def evaluator(m, target_metric, **kw):
        t = tuple(int(x) for x in m.mlrank)
        visited.append(t)
        res[prefix + "lists_" + _key(t)] = np.array(m.recommendations, dtype=np.int64)
        res[prefix + "item_" + _key(t)] = np.asarray(m.factors[f.itemid], dtype=np.float64)
        res[prefix + "fdbk_" + _key(t)] = np.asarray(m.factors[f.feedback], dtype=np.float64)
        return evaluate_models(m, target_metric, **kw)

    best, scores = find_optimal_tucker_ranks(model, mlranks, "recall", return_scores=True, same_space=same_space,
                                             evaluator=evaluator, metric_type="relevance")
    idx, val, shp = data.to_coo(tensor_mode=True)
    (tu, ti, tf), tshape, tusers = model._get_test_data()
    h = data.test.holdout
    res.update({prefix + k: v for k, v in dict(
        train_idx=idx.astype(np.int64), train_val=val.astype(np.float64), train_shape=np.array(shp),
        test_user=tu.astype(np.int64), test_item=ti.astype(np.int64), test_fdbk=np.asarray(tf, dtype=np.int64),
        test_shape=np.array(tshape), holdout_user=h[f.userid].values.astype(np.int64),
        holdout_item=h[f.itemid].values.astype(np.int64), holdout_fdbk=h[f.feedback].values.astype(np.float64),
        topk=np.array(model.topk), n_items=np.array(data.index.itemid.shape[0]),
        switch_positive=np.array(np.nan if model.switch_positive is None else model.switch_positive),
        ranks_r1=np.array(mlranks[0]), ranks_r2=np.array(mlranks[1]), ranks_r3=np.array(mlranks[2]),
        same_space=np.array(same_space), flattener=np.array(-1 if flattener is None else flattener),
        mlrank=np.array(model.mlrank), u0=model.factors[f.userid], u1=model.factors[f.itemid],
        u2=model.factors[f.feedback], core=model.factors["core"], visited=np.array(visited, dtype=np.int64),
        score_index=np.array(list(scores.index), dtype=np.int64), scores=scores.values.astype(np.float64),
        best=np.array(best, dtype=np.int64)).items()})
    print(prefix, "built", model.mlrank, "visited", len(visited), "best", best, "scores", scores.round(4).to_dict())


def main():
    import_reference()
    res = {}
    case(res, "a_", 11, ([10, 6, 2], [8, 5, 2], [4, 3, 1]), False)
    case(res, "b_", 12, ([8, 5, 3], [8, 5, 3], [4, 2]), True, flattener=[2, 3])
    np.savez_compressed(OUT, **res)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

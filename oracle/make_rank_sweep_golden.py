"""Generate ``tests/golden/rank_sweep.npz`` by running the REAL reference's rank search
(``polara.evaluation.pipelines.find_optimal_svd_rank``, pipelines.py:81-116).  TEST INFRASTRUCTURE; needs numba and the
reference checkout named by POLARA_REFERENCE_ROOT.

    POLARA_REFERENCE_ROOT=... python oracle/make_rank_sweep_golden.py

The search is given an ``evaluator`` that wraps the reference's ``evaluate_models`` (pipelines.py:63-78) and records
``model.recommendations`` at each rank, so the fixture holds the lists the metrics were computed from.  Two cases:

* ``s_*`` -- sampled evaluation, drawn on the fly: the data model of ``make_sampler_golden.model_run``
  (``planted_ratings(700, 420, 40, rank=6, seed=21)``, ``seed=5``, holdout 1, 99 unseen items) under
  ``RandomSampleEvaluationSVDMixin``; built at rank 12, ranks (12, 10, 8, 6, 4, 2, 1), target ``mrr`` with
  ``metric_type='ranking'`` and ``simple_rates=True``.  The reference's ``evaluate()`` for this model matches the lists
  against the holdout column ``x_<itemid>`` (data.py:945-962), which only ``set_unseen_interactions`` adds; with the
  draw made on the fly nothing calls it, so this maker calls ``data.adapt_holdout()`` itself.
* ``k_*`` -- standard protocol: a plain ``SVDModel`` on a known-user split (``warm_start = False``), ranks
  (16, 12, 8, 5, 3, 1), target ``recall`` with ``metric_type='relevance'`` (precision and nDCG are avoided: the
  reference's ``safe_divide`` leaves masked entries uninitialised).

Stored per case: the inputs the model reads (test triplets and shape, holdout columns), the item factors at the build
rank, the lists at each rank (``<case>_lists_r<rank>``), the score Series (values in the order of ``ranks``) and the best
rank.
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

OUT = os.path.join(ROOT, "tests", "golden", "rank_sweep.npz")


def _search(model, ranks, target, **kwargs):
    """find_optimal_svd_rank with an evaluator that records the lists behind every score."""
    from polara.evaluation.pipelines import evaluate_models, find_optimal_svd_rank
    lists = {}

    def evaluator(m, target_metric, **kw):
        res = evaluate_models(m, target_metric, **kw)
        lists[m.rank] = np.array(m.recommendations, dtype=np.int64)
        return res
    best, scores = find_optimal_svd_rank(model, ranks, target, return_scores=True, evaluator=evaluator, **kwargs)
    return best, scores, lists


def _store(res, prefix, model, ranks, best, scores, lists, extra):
    f = model.data.fields
    (tu, ti, tf), tshape, _ = model._get_test_data()
    res.update({prefix + "test_user": np.asarray(tu, np.int64), prefix + "test_item": np.asarray(ti, np.int64),
                prefix + "test_fdbk": np.asarray(tf, np.float64), prefix + "shape": np.array(tshape, np.int64),
                prefix + "item_factors": model.factors[f.itemid], prefix + "ranks": np.array(ranks, np.int64),
                prefix + "scores": scores.loc[list(ranks)].values.astype(np.float64), prefix + "best": np.array(best),
                prefix + "topk": np.array(model.topk), prefix + "n_items": np.array(model.data.index.itemid.shape[0])})
    for r, lst in lists.items():
        res[prefix + "lists_r%d" % r] = lst
    res.update({prefix + k: v for k, v in extra.items()})
    print(prefix, "best rank", best, dict(zip(ranks, scores.loc[list(ranks)].round(5))))


def sampled_case(res):
    from polara.recommender.data import RecommenderData, RandomSampleEvaluationMixin
    from polara.recommender.models import RandomSampleEvaluationSVDMixin, SVDModel

    class SampledData(RandomSampleEvaluationMixin, RecommenderData):
        pass

    class SampledSVD(RandomSampleEvaluationSVDMixin, SVDModel):
        pass

    u, i, r = planted_ratings(700, 420, 40, rank=6, seed=21)
    data = SampledData(pd.DataFrame({"userid": u, "itemid": i, "rating": r}), "userid", "itemid", "rating", seed=5)
    data.holdout_size = 1
    data.warm_start = False
    data.verbose = False
    data.prepare()
    data.unseen_items_num = 99
    data.adapt_holdout()                      # the x_<itemid> column evaluate() reads (see the module docstring)
    model = SampledSVD(data)
    model.verbose = False
    model.rank = 12
    model.topk = 10
    ranks = [12, 10, 8, 6, 4, 2, 1]
    best, scores, lists = _search(model, ranks, "mrr", metric_type="ranking", simple_rates=True)
    hold = data.test.holdout
    f = data.fields
    _store(res, "s_", model, ranks, best, scores, lists,
           dict(holdout_user=hold[f.userid].values.astype(np.int64), holdout_item=hold[f.itemid].values.astype(np.int64),
                holdout_pos=hold["x_" + f.itemid].values.astype(np.int64), n_unseen=np.array(99),
                data_seed=np.array(data.seed)))


def standard_case(res):
    from polara.recommender.data import RecommenderData
    from polara.recommender.models import SVDModel
    u, i, r = planted_ratings(600, 380, 36, rank=6, seed=13)
    data = RecommenderData(pd.DataFrame({"userid": u, "itemid": i, "rating": r}), "userid", "itemid", "rating", seed=3)
    data.warm_start = False
    data.verbose = False
    data.prepare()
    model = SVDModel(data)
    model.verbose = False
    model.rank = 16
    model.topk = 10
    ranks = [16, 12, 8, 5, 3, 1]
    best, scores, lists = _search(model, ranks, "recall", metric_type="relevance")
    hold = data.test.holdout
    f = data.fields
    _store(res, "k_", model, ranks, best, scores, lists,
           dict(holdout_user=hold[f.userid].values.astype(np.int64), holdout_item=hold[f.itemid].values.astype(np.int64),
                holdout_fdbk=hold[f.feedback].values.astype(np.float64)))


def main():
    import_reference()
    res = {}
    sampled_case(res)
    standard_case(res)
    np.savez_compressed(OUT, **res)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

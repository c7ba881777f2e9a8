"""Generate ``tests/golden/sampler_cases.npz`` by running the REAL reference's sampler (polara/lib/sampler.py) and its
on-the-fly sampled evaluation (RandomSampleEvaluationSVDMixin.get_recommendations, models.py:1137-1183).  TEST
INFRASTRUCTURE; needs numba and the reference checkout named by POLARA_REFERENCE_ROOT.

    POLARA_REFERENCE_ROOT=... python oracle/make_sampler_golden.py

Stored per ``sample_row_wise`` case ``c<j>_*``: n (item count), s (samples per row), indptr / indices (exclusion lists in
the order the reference reads them), seeds (uint32) and out (the reference's draw).  ``mf_*``: one
``mf_random_item_scoring`` call on case 0's lists.  ``run_*``: one full model run (see :func:`model_run`).
"""
import os
import sys

import numpy as np
import pandas as pd
import scipy.sparse as sps

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.ref_shim import import_reference  # noqa: E402
from polara_b200.synth import planted_ratings  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "sampler_cases.npz")


def _csr(lists):
    indptr = np.zeros(len(lists) + 1, dtype=np.int64)
    indptr[1:] = np.cumsum([len(x) for x in lists])
    indices = np.concatenate([np.asarray(x, dtype=np.int32) for x in lists]) if lists else np.empty(0, np.int32)
    return indptr, indices.astype(np.int32)


def _scipy_general_order(rng, n, n_rows):
    """rows of ``profile + holdout`` where the holdout rows are unsorted: scipy's non-canonical add decides the order."""
    prof = []
    hold = []
    for _ in range(n_rows):
        items = rng.choice(n, int(rng.integers(3, 25)), replace=False)
        cut = int(rng.integers(1, 3))
        prof.append(np.sort(items[cut:]))
        hold.append(items[:cut][::-1] if cut > 1 and items[0] < items[1] else items[:cut])
    p_ptr, p_idx = _csr(prof)
    h_ptr, h_idx = _csr(hold)
    p = sps.csr_matrix((np.ones(len(p_idx)), p_idx, p_ptr), shape=(n_rows, n)).copy()
    h = sps.csr_matrix((n_rows, n), dtype=bool)
    h.data, h.indices, h.indptr = np.ones(len(h_idx), dtype=bool), h_idx, h_ptr
    s = p + h
    return [s.indices[s.indptr[r]:s.indptr[r + 1]].copy() for r in range(n_rows)]


def cases():
    rng = np.random.default_rng(2024)
    out = []
    # case 0: n = 300, 50 samples; every adversarial list shape
    n, s = 300, 50
    lists = []
    for _ in range(6):
        lists.append(np.sort(rng.choice(n, int(rng.integers(5, 60)), replace=False)))          # sorted
    for _ in range(6):
        lists.append(np.sort(rng.choice(n, int(rng.integers(5, 60)), replace=False))[::-1])    # reversed
    lists += _scipy_general_order(rng, n, 8)                                                   # scipy general path
    for _ in range(6):                                                                         # items in the tail
        m = int(rng.integers(10, 80))
        tail = rng.choice(np.arange(n - m, n), int(rng.integers(1, m)), replace=False)
        head = rng.choice(n - m, m - len(tail), replace=False)
        x = np.concatenate([tail, head, [n - 1]] if n - 1 not in tail else [tail, head])
        rng.shuffle(x)
        lists.append(x)
    lists.append(np.array([], dtype=np.int32))                                                 # empty
    lists.append(np.array([n - 1]))
    lists.append(rng.permutation(n)[: n - s])                                                  # exactly s left
    lists.append(np.sort(rng.choice(n, n - s, replace=False))[::-1])
    while len(lists) < 40:
        lists.append(rng.permutation(n)[: int(rng.integers(0, 120))])
    seeds = np.random.SeedSequence(0).generate_state(len(lists))
    seeds[0], seeds[1] = 0, 2 ** 32 - 1
    out.append((n, s, lists, seeds))
    # case 1: one sample per row
    n = 97
    lists = [rng.permutation(n)[: int(rng.integers(0, 96))] for _ in range(24)]
    out.append((n, 1, lists, np.random.SeedSequence(1).generate_state(len(lists))))
    # cases 2..: n = 2^j and 2^j +- 1, remaining crossing powers of two while it shrinks
    for j, n in enumerate((255, 256, 257, 1023, 1024, 1025, 4096)):
        s = min(n - 40, 600)
        lists = [np.array([], dtype=np.int32), np.array([n - 1, 0]), rng.permutation(n)[:40],
                 np.sort(rng.permutation(n)[:17])[::-1], rng.permutation(n)[: n - s]]
        seeds = np.random.SeedSequence(10 + j).generate_state(len(lists))
        seeds[-1] = 2 ** 32 - 1
        out.append((n, s, lists, seeds))
    return out


def model_run(res):
    """One on-the-fly ``get_recommendations`` of RandomSampleEvaluationSVDMixin on a seeded data model."""
    from polara.recommender.data import RecommenderData, RandomSampleEvaluationMixin
    from polara.recommender.models import RandomSampleEvaluationSVDMixin, SVDModel
    from polara.recommender.evaluation import matrix_from_observations
    from polara.lib.sampler import sample_row_wise

    class SampledData(RandomSampleEvaluationMixin, RecommenderData):
        pass

    class SampledSVD(RandomSampleEvaluationSVDMixin, SVDModel):
        pass

    u, i, r = planted_ratings(700, 420, 40, rank=6, seed=21)
    df = pd.DataFrame({"userid": u, "itemid": i, "rating": r})
    data = SampledData(df, "userid", "itemid", "rating", seed=5)
    data.holdout_size = 1
    data.warm_start = False
    data.verbose = False
    data.prepare()
    data.unseen_items_num = 99
    model = SampledSVD(data)
    model.verbose = False
    model.rank = 12
    model.topk = 10
    model.build()
    pos = model.get_recommendations()
    f = data.fields
    (tu, ti, tf), tshape, _ = model._get_test_data()
    test_matrix, _ = model.get_test_matrix()
    holdout = data.test.holdout
    hm = matrix_from_observations(holdout, f.userid, f.itemid, test_matrix.shape, feedback=None)
    all_seen = test_matrix + hm
    seeds = np.random.SeedSequence(data.seed).generate_state(test_matrix.shape[0])
    sampled = sample_row_wise(all_seen.indptr, all_seen.indices, test_matrix.shape[1], 99, seeds)
    v = model.factors[f.itemid]
    e = test_matrix.dot(v)
    res.update(run_test_user=np.asarray(tu, np.int64), run_test_item=np.asarray(ti, np.int64),
               run_test_fdbk=np.asarray(tf, np.float64), run_shape=np.array(tshape, dtype=np.int64),
               run_holdout_user=holdout[f.userid].values.astype(np.int64),
               run_holdout_item=holdout[f.itemid].values.astype(np.int64),
               run_item_factors=v, run_excl_indptr=all_seen.indptr.astype(np.int64),
               run_excl_indices=all_seen.indices.astype(np.int32), run_seeds=seeds, run_sampled=sampled.astype(np.int32),
               run_unseen_scores=model.compute_random_item_scores_gen(e, v, test_matrix, 99),
               run_positions=pos.astype(np.int64), run_topk=np.array(model.topk), run_n_unseen=np.array(99),
               run_data_seed=np.array(data.seed))
    print("model run: users", tshape[0], "items", tshape[1], "positions", pos.shape)


def main():
    import_reference()
    from polara.lib.sampler import mf_random_item_scoring, sample_row_wise
    import numba
    res = {}
    for j, (n, s, lists, seeds) in enumerate(cases()):
        indptr, indices = _csr(lists)
        drawn = sample_row_wise(indptr, indices, n, s, seeds)
        res.update({"c%d_n" % j: np.array(n), "c%d_s" % j: np.array(s), "c%d_indptr" % j: indptr,
                    "c%d_indices" % j: indices, "c%d_seeds" % j: seeds.astype(np.uint32), "c%d_out" % j: drawn})
    res["n_cases"] = np.array(j + 1)
    # mf_random_item_scoring on case 0: scores of the items it draws (the same draw as sample_row_wise)
    n, s = int(res["c0_n"]), int(res["c0_s"])
    rng = np.random.default_rng(7)
    uf = rng.standard_normal((len(res["c0_indptr"]) - 1, 8))
    vf = rng.standard_normal((n, 8))
    scores = np.zeros((uf.shape[0], s))
    mf_random_item_scoring(uf, vf, res["c0_indptr"], res["c0_indices"], s, res["c0_seeds"], scores)
    res.update(mf_user_factors=uf, mf_item_factors=vf, mf_scores=scores)
    model_run(res)
    res["numba_threads"] = np.array(numba.get_num_threads())
    np.savez_compressed(OUT, **res)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

"""Item cold start at the MovieLens-20M shape: the device build of B200SVDModelItemColdStart, its cold scoring call and
``evaluate()``, and the fused scoring kernel at the standard shape for comparison.

    python scripts/coldstart_bench.py [--reps 3] [--rank 50] [--no-reference] [--out FILE]

Synthetic data from ``polara_b200.synth.popularity_csr``: 138 493 users x 26 744 items, 20 M draws; 20 % of the items
(seeded) are cold and all their interactions form the holdout, the rest is the training matrix.  Every item has 1-3 of
20 genre-like labels.  Times: the build (``model.build()``: the device SVD with U, then W = F^T V and pinv(W^T W) on the
host) and ``evaluate()`` on the host clock after a synchronisation; the cold scoring call (``get_recommendations()``:
F_cold (W pinv(W^T W)) on the device and the top-10 users of every cold item) with CUDA events; medians, min and max over
``--reps`` calls after one warm-up.  ``standard_score`` times the same fused kernel at the standard shape, 20 % of the
users against the training items, for the pairs/s comparison.  The reference's host SVDModelItemColdStart (from
oracle/_ref, with a stub ``lightfm``) is timed where it is installed, unless ``--no-reference``.  Prints one JSON line
with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from i2i_bench import card, timed  # noqa: E402

N_USERS, N_ITEMS, NNZ = 138_493, 26_744, 20_000_000
N_LABELS = 20


def make_problem(seed=3):
    """``(train_idx, train_val, train_shape, cold arrays, F, F_cold, item labels, cold ids)`` of the synthetic split."""
    import scipy.sparse as sps
    from polara_b200.synth import popularity_csr
    indptr, indices, values = popularity_csr(N_USERS, N_ITEMS, NNZ, seed=seed)
    rng = np.random.default_rng(seed + 1)
    cold = np.zeros(N_ITEMS, dtype=bool)
    cold[rng.permutation(N_ITEMS)[:N_ITEMS // 5]] = True
    new_id = np.empty(N_ITEMS, dtype=np.int64)
    new_id[~cold] = np.arange((~cold).sum())
    new_id[cold] = np.arange(cold.sum())
    user = np.repeat(np.arange(N_USERS, dtype=np.int64), np.diff(indptr))
    item = np.asarray(indices, dtype=np.int64)
    val = np.asarray(values, dtype=np.float64)
    is_cold = cold[item]
    train_idx = np.stack([user[~is_cold], new_id[item[~is_cold]]], axis=1)
    n_train = int((~cold).sum())
    labels = [rng.choice(N_LABELS, rng.integers(1, 4), replace=False) for _ in range(N_ITEMS)]
    rows = np.repeat(np.arange(N_ITEMS), [len(x) for x in labels])
    onehot = sps.csr_matrix((np.ones(len(rows)), (rows, np.concatenate(labels))), shape=(N_ITEMS, N_LABELS))
    order_train, order_cold = np.flatnonzero(~cold), np.flatnonzero(cold)
    return dict(train_idx=train_idx, train_val=val[~is_cold], train_shape=(N_USERS, n_train),
                cold_item=new_id[item[is_cold]], cold_user=user[is_cold], cold_fdbk=val[is_cold],
                f=onehot[order_train], f_cold=onehot[order_cold], labels=labels, cold_orig=order_cold,
                train_orig=order_train)


def host_clock(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    s = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        s.append((time.perf_counter() - t0) * 1e3)
    return dict(median_ms=float(np.median(s)), min_ms=float(np.min(s)), max_ms=float(np.max(s)))


def reference_times(pb, rank):
    """the reference's SVDModelItemColdStart on ItemColdStartData of the same split: build and get_recommendations."""
    import types
    from oracle import ref_driver as rd
    if rd.reference_root() is None:
        return None
    rd.import_reference()
    import pandas as pd
    sys.modules.setdefault("lightfm", types.SimpleNamespace(LightFM=object))
    from polara.recommender.coldstart.data import ItemColdStartData
    from polara.recommender.coldstart.models import SVDModelItemColdStart
    orig_item = np.r_[pb["train_orig"][pb["train_idx"][:, 1]], pb["cold_orig"][pb["cold_item"]]]
    frame = pd.DataFrame({"userid": np.r_[pb["train_idx"][:, 0], pb["cold_user"]], "itemid": orig_item,
                          "rating": np.r_[pb["train_val"], pb["cold_fdbk"]]})
    feats = pd.DataFrame({"genres": [list(x) for x in pb["labels"]]})
    data = ItemColdStartData(frame, "userid", "itemid", "rating", seed=1, item_features=feats)
    data.verbose = False
    data.prepare()
    model = SVDModelItemColdStart(data)
    model.verbose = False
    model.rank = rank
    t0 = time.perf_counter()
    model.build()
    t1 = time.perf_counter()
    model.get_recommendations()
    t2 = time.perf_counter()
    return dict(build_s=t1 - t0, score_s=t2 - t1, cold_items=int(data.index.itemid.cold_start.shape[0]),
                note="the reference's own split (seed 1) of the same interactions, one run each")


def run(reps, rank, reference):
    import torch
    from polara_b200.engine import round_up
    from polara_b200.host import ColdStartData
    from polara_b200.models import B200SVDModelItemColdStart
    pb = make_problem()
    data = ColdStartData(pb["train_idx"], pb["train_val"], pb["train_shape"], pb["cold_item"], pb["cold_user"],
                         pb["cold_fdbk"], pb["f"], pb["f_cold"], n_users=N_USERS)
    model = B200SVDModelItemColdStart(data)
    model.verbose = False
    model.rank = rank
    model.topk = 10
    n_cold = int(data.index.itemid.cold_start.shape[0])
    rec = dict(users=N_USERS, items=N_ITEMS, train_items=int(pb["train_shape"][1]), train_nnz=int(len(pb["train_val"])),
               cold_items=n_cold, holdout_rows=int(len(data.test.holdout)), rank=rank, topk=10, card=card())
    rec["build"] = host_clock(model.build, reps)
    rec["cold_score"] = timed(model.get_recommendations, reps)
    rec["cold_pairs_per_s"] = n_cold * N_USERS / (rec["cold_score"]["median_ms"] * 1e-3)

    def evaluate():
        model._recommendations = None
        model._recommendations = model.get_recommendations()
        t0 = time.perf_counter()
        model.evaluate()
        return time.perf_counter() - t0
    evaluate()
    rec["evaluate_ms"] = float(np.median([evaluate() * 1e3 for _ in range(reps)]))
    # the fused kernel at the standard shape: every 5th user's U diag(s) row against the training items' V
    eng = model.engine
    ld = round_up(rank, 32)
    u = model.factors["userid"][::5] * model.factors["singular_values"][None, :]
    e = np.zeros((u.shape[0], ld), np.float32)
    e[:, :rank] = u
    v = np.zeros((model.factors["itemid"].shape[0], ld), np.float32)
    v[:, :rank] = model.factors["itemid"]
    e_dev, v_dev = eng.upload(e), eng.upload(v)
    rec["standard_score"] = timed(lambda: eng.score_topk(e_dev, v_dev, rank, 10), reps)
    rec["standard_pairs_per_s"] = u.shape[0] * v.shape[0] / (rec["standard_score"]["median_ms"] * 1e-3)
    del e_dev, v_dev
    torch.cuda.empty_cache()
    rec["reference"] = reference_times(pb, rank) if reference else "not measured (--no-reference)"
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--rank", type=int, default=50)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    line = json.dumps(run(args.reps, args.rank, not args.no_reference))
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

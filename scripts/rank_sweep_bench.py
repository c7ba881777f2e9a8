"""Timing of the rank sweep of find_optimal_svd_rank (ranks 10, 20, ..., 150, top-10, 1 holdout + 999 sampled unseen
items per user on the sampled protocol): one sweep against the per-rank loop it replaces.

    python scripts/rank_sweep_bench.py [--reps 3] [--large-reps 2] [--large-users 1000000] [--only eigenrec|large]

Two workloads, the data of scripts/sampled_eval_bench.py: EIGENREC-sized (3140 users x 3706 items, ~165 items per
profile) and C2-sized (1 M users x 100 K items, 1e8 nnz, polara_b200.synth.popularity_csr), item factors of width 150.
Per workload, one JSON line with, as median / min / max over the repetitions (host clock around work that ends in a
copy to the host):
  * sampled_model_ms: the per-rank loop (model.rank = r; sampled_recommendations, ranks descending as
    find_optimal_svd_rank walks them) against one sampled_rank_sweep;
  * sampled_device_ms: R x Engine.sampled_topk on one E_max against one Engine.sampled_topk_ranks (CUDA events);
  * standard_model_ms (C2 only): the per-rank get_recommendations loop against one rank_sweep;
plus flags: whether the sweep's lists equal the single-rank calls on E_max bit for bit, and the share of list entries
the sweep has in common with the per-rank model loop (that loop forms E at each rank, see DESIGN.md section 4).
The device name and its power limit are read in the same run.  Writes nothing but stdout, and a progress line per
phase to stderr.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

RANKS = list(range(10, 151, 10))
N_UNSEEN = 999
TOPK = 10


def _progress(msg):
    print("rank_sweep_bench: " + msg, file=sys.stderr, flush=True)


def _stats(xs):
    return {"median": float(np.median(xs)), "min": float(min(xs)), "max": float(max(xs)), "reps": len(xs)}


def _host_ms(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def _event_ms(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def run(name, n_users, n_items, nnz, reps, standard, seed=1):
    from polara_b200.engine import get_engine
    from polara_b200.host import ArrayData
    from polara_b200.models import B200SVDModel, sampled_exclusion_lists
    from sampled_eval_bench import card, workload
    eng = get_engine(0)
    user, item, fdbk, hold = workload(n_users, n_items, nnz, seed)
    shape = (n_users, n_items)
    width = RANKS[-1]
    rng = np.random.default_rng(seed + 2)
    v = rng.standard_normal((n_items, width)) / np.sqrt(width)
    data = ArrayData(np.zeros((1, 2), dtype=np.int64), np.ones(1), shape, user, item, fdbk, shape, warm_start=False)
    model = B200SVDModel(data)
    model.verbose = False
    model.rank = width
    model.topk = TOPK
    full = {"userid": None, "itemid": v, "singular_values": np.ones(width)}
    hold2 = hold.reshape(-1, 1)

    def reset():
        model._rank = width
        model.factors = dict(full)
        model._recommendations = None

    def sampled_loop():
        out = {}
        for r in sorted(RANKS, reverse=True):
            model.rank = r
            out[r] = model.sampled_recommendations(hold2, None, n_unseen=N_UNSEEN, seed=seed)
        reset()
        return out

    def sampled_sweep():
        return model.sampled_rank_sweep(RANKS, hold2, n_unseen=N_UNSEEN, seed=seed)

    res = {"workload": name, "users": n_users, "items": n_items, "profile_nnz": int(len(user)), "ranks": RANKS,
           "topk": TOPK, "holdout": 1, "n_unseen": N_UNSEEN}
    _progress("%s: sampled protocol through the model" % name)
    reset()
    sampled_sweep()                                                         # warm-up of every kernel on the path
    loop_ms, sweep_ms = [], []
    for _ in range(reps):
        t, loop_lists = _host_ms(sampled_loop)
        loop_ms.append(t)
        t, sweep_lists = _host_ms(sampled_sweep)
        sweep_ms.append(t)
    res["sampled_model_ms"] = {"per_rank_loop": _stats(loop_ms), "sweep": _stats(sweep_ms)}
    res["sampled_model_agreement_with_loop"] = float(np.mean([(sweep_lists[r] == loop_lists[r]).mean() for r in RANKS]))

    _progress("%s: sampled protocol, device calls" % name)
    # the device calls alone, on one E_max and the test data the model reads
    test_data = model._get_test_data()[0]
    p_dev, _ = model._test_csr_device(test_data, shape)
    v_dev = model._device_factor("itemid")
    e = eng.spmm(p_dev, v_dev, ell=width)
    indptr, indices = sampled_exclusion_lists(test_data, shape, hold2)
    ip, ix, hd = eng.upload(indptr), eng.upload(indices), eng.upload(hold2)
    sd = eng.upload(np.ascontiguousarray(np.random.SeedSequence(seed).generate_state(n_users)).view(np.int32))

    def singles():
        return [eng.sampled_topk(e, v_dev, r, hd, ip, ix, sd, N_UNSEEN, TOPK) for r in RANKS]

    def multi():
        return eng.sampled_topk_ranks(e, v_dev, RANKS, hd, ip, ix, sd, N_UNSEEN, TOPK)
    singles()
    multi()
    single_ms, multi_ms = [], []
    for _ in range(reps):
        t, one = _event_ms(singles)
        single_ms.append(t)
        t, many = _event_ms(multi)
        multi_ms.append(t)
    res["sampled_device_ms"] = {"single_rank_calls": _stats(single_ms), "multi_rank_call": _stats(multi_ms)}
    res["sampled_sweep_equals_single_rank_calls"] = bool(all(
        np.array_equal(many[j].cpu().numpy(), one[j].cpu().numpy()) for j in range(len(RANKS))))
    res["sampled_model_sweep_equals_device_call"] = bool(all(
        np.array_equal(sweep_lists[r], many[j].cpu().numpy()) for j, r in enumerate(RANKS)))
    del p_dev, e, ip, ix, hd, one, many

    if standard:
        _progress("%s: standard protocol" % name)

        def standard_loop():
            out = {}
            for r in sorted(RANKS, reverse=True):
                model.rank = r
                out[r] = model.get_recommendations()
            reset()
            return out

        def standard_sweep():
            return model.rank_sweep(RANKS)
        standard_sweep()
        standard_loop()
        loop_ms, sweep_ms = [], []
        for _ in range(reps):
            t, loop_lists = _host_ms(standard_loop)
            loop_ms.append(t)
            t, sweep_lists = _host_ms(standard_sweep)
            sweep_ms.append(t)
        res["standard_model_ms"] = {"per_rank_loop": _stats(loop_ms), "sweep": _stats(sweep_ms)}
        res["standard_agreement_with_loop"] = float(np.mean([(sweep_lists[r] == loop_lists[r]).mean() for r in RANKS]))
        # the sweep against the fused kernel on the same E_max, rank by rank
        big = model._big_test_triplets()
        p_dev, seen = model._test_csr_device(big[0] if big else model._get_test_data()[0], shape)
        e = eng.spmm(p_dev, v_dev, ell=v_dev.shape[1])
        res["standard_sweep_equals_single_rank_calls"] = bool(all(
            np.array_equal(sweep_lists[r], eng.score_topk(e, v_dev, r, TOPK, seen=seen).cpu().numpy()) for r in RANKS))
    res.update(card())
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--large-reps", type=int, default=2)
    ap.add_argument("--large-users", type=int, default=1_000_000)
    ap.add_argument("--large-nnz", type=int, default=100_000_000)
    ap.add_argument("--only", choices=["eigenrec", "large"], default=None)
    args = ap.parse_args()
    if args.only in (None, "eigenrec"):
        run("eigenrec", 3140, 3706, 3140 * 165, args.reps, standard=False)
    if args.only in (None, "large"):
        run("large_c2", args.large_users, 100_000, args.large_nnz, args.large_reps, standard=True)


if __name__ == "__main__":
    main()

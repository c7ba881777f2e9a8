"""Timing of the on-the-fly sampled evaluation (1 holdout + 999 sampled unseen items per user, rank 50).

    python scripts/sampled_eval_bench.py [--large-users 1000000] [--reps 5] [--ref-users 20000]

Two workloads: EIGENREC-sized (3140 users x 3706 items, ~165 items per profile) and large (1 M users x 100 K items, C2
data from polara_b200.synth.popularity_csr, 100 M nnz).  Per workload, one JSON line with:
  * fused_ms: pb200_sampled_topk (check pass + draw/score/rank kernel), CUDA events, after a warm-up call, over --reps
    calls: median, min, max;
  * exclusion_ms: the host construction of the exclusion lists (scipy profile + holdout, as the reference does);
  * end_to_end_ms: B200SVDModel.sampled_recommendations (test CSR ingest, SpMM, exclusion lists, fused call, copy back);
  * reference_ms: the reference's mf_random_item_scoring (numba, parallel) on the first --ref-users users, with the numba
    thread count, extrapolated linearly to all users and labelled so; "not run" without a reference under oracle/_ref.
The device name and its power limit are read in the same run.  Writes nothing but stdout.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    out = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit"] = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        out["power_limit"] = "unknown"
    return out


def workload(n_users, n_items, nnz, seed):
    """profile CSR (holdout removed), one holdout item per user (a random one of the user's items), test triplets."""
    from polara_b200.synth import popularity_csr
    indptr, indices, data = popularity_csr(n_users, n_items, nnz, seed=seed)
    rng = np.random.default_rng(seed + 1)
    lens = np.diff(indptr)
    pick = indptr[:-1] + (rng.random(n_users) * lens).astype(np.int64)          # every row has >= 1 item
    hold = indices[pick].astype(np.int64)
    keep = np.ones(len(indices), bool)
    keep[pick] = False
    user = np.repeat(np.arange(n_users, dtype=np.int64), lens)[keep]
    item = indices[keep].astype(np.int64)
    fdbk = data[keep].astype(np.float64)
    return user, item, fdbk, hold


def run(name, n_users, n_items, nnz, rank, n_unseen, reps, ref_users, seed=1):
    import torch
    from polara_b200.engine import get_engine
    from polara_b200.host import ArrayData
    from polara_b200.models import B200SVDModel, sampled_exclusion_lists
    eng = get_engine(0)
    user, item, fdbk, hold = workload(n_users, n_items, nnz, seed)
    shape = (n_users, n_items)
    rng = np.random.default_rng(seed + 2)
    v = (rng.standard_normal((n_items, rank)) / np.sqrt(rank)).astype(np.float32)
    data = ArrayData(np.zeros((1, 2), dtype=np.int64), np.ones(1), shape, user, item, fdbk, shape, warm_start=False)
    model = B200SVDModel(data)
    model.verbose = False
    model.rank = rank
    model.topk = 10
    model.factors = {"userid": None, "itemid": v, "singular_values": np.ones(rank)}
    model._is_ready = True
    hold2 = hold.reshape(-1, 1)
    # exclusion lists (host) and the device call alone
    t0 = time.perf_counter()
    indptr, indices = sampled_exclusion_lists((user, item, fdbk), shape, hold2)
    excl_ms = (time.perf_counter() - t0) * 1e3
    seeds = np.random.SeedSequence(seed).generate_state(n_users)
    p_dev, _ = model._test_csr_device((user, item, fdbk), shape)
    v_dev = model._device_factor("itemid")
    e = eng.spmm(p_dev, v_dev, ell=rank)
    ip, ix, hd = eng.upload(indptr), eng.upload(indices), eng.upload(hold2)
    sd = eng.upload(np.ascontiguousarray(seeds).view(np.int32))
    eng.sampled_topk(e, v_dev, rank, hd, ip, ix, sd, n_unseen, 10)                   # warm-up
    stats = eng.sampler_stats()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        eng.sampled_topk(e, v_dev, rank, hd, ip, ix, sd, n_unseen, 10)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    # end to end through the model
    model.sampled_recommendations(hold2, None, n_unseen=n_unseen, seed=seed)          # warm-up
    e2e = []
    for _ in range(max(1, reps // 2)):
        t0 = time.perf_counter()
        model.sampled_recommendations(hold2, None, n_unseen=n_unseen, seed=seed)
        e2e.append((time.perf_counter() - t0) * 1e3)
    res = {"workload": name, "users": n_users, "items": n_items, "profile_nnz": int(len(user)),
           "exclusion_nnz": int(len(indices)), "rank": rank, "holdout": 1, "n_unseen": n_unseen,
           "fused_ms": {"median": float(np.median(times)), "min": float(min(times)), "max": float(max(times)),
                        "reps": reps},
           "map_paths": stats, "exclusion_ms": excl_ms,
           "end_to_end_ms": {"median": float(np.median(e2e)), "min": float(min(e2e)), "max": float(max(e2e)),
                             "reps": len(e2e)},
           "end_to_end_exclusion_ms": model.last_sampled_timings["exclusion_ms"]}
    res["reference_ms"] = reference_time(e, indptr, indices, seeds, v, rank, n_unseen, ref_users)
    res.update(card())
    print(json.dumps(res), flush=True)


def reference_time(e, indptr, indices, seeds, v, rank, n_unseen, ref_users):
    """the reference's numba kernel on the first ref_users users, extrapolated to all of them."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "polara")):
        return "not run (no reference under oracle/_ref)"
    sys.path.insert(0, ref)
    try:
        import numba
        from polara.lib.sampler import mf_random_item_scoring
    except ImportError as exc:
        return "not run (%s)" % exc
    m = len(indptr) - 1
    sub = min(m, ref_users)
    uf = e[:sub, :rank].cpu().numpy().astype(np.float64)
    vf = v.astype(np.float64)
    ip = indptr[:sub + 1]
    ix = indices[:ip[-1]]
    res = np.zeros((2, n_unseen))
    mf_random_item_scoring(uf[:2], vf, ip[:3], ix[:ip[2]], n_unseen, seeds[:2], res)   # JIT compile
    res = np.zeros((sub, n_unseen))
    t0 = time.perf_counter()
    mf_random_item_scoring(uf, vf, ip, ix, n_unseen, seeds[:sub], res)
    ms = (time.perf_counter() - t0) * 1e3
    return {"measured_users": sub, "measured_ms": ms, "numba_threads": int(numba.get_num_threads()),
            "all_users_ms_extrapolated": ms * m / sub}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--large-users", type=int, default=1_000_000)
    ap.add_argument("--large-nnz", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-users", type=int, default=20_000)
    ap.add_argument("--only", choices=["eigenrec", "large"], default=None)
    args = ap.parse_args()
    from polara_b200 import _build
    _build.build()
    if args.only in (None, "eigenrec"):
        run("eigenrec", 3140, 3706, 3140 * 165, 50, 999, args.reps, args.ref_users)
    if args.only in (None, "large"):
        run("large_c2", args.large_users, 100_000, args.large_nnz, 50, 999, args.reps, args.ref_users)


if __name__ == "__main__":
    main()

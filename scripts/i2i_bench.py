"""Item-to-item model (CooccurrenceModel) on the device: build and scoring time at MovieLens-1M and MovieLens-20M shapes.

    python scripts/i2i_bench.py [--shapes ml1m,ml20m] [--reps 5] [--ref-users-ml20m 300] [--out FILE]

Synthetic data from ``polara_b200.synth.popularity_csr``.  The training matrix is every user; the test matrix is the
profile of every ``--test-every``-th user (the test profiles are what the scoring multiplies by S).  Times are CUDA
events around ``Engine.cooc_build`` (transpose, panel split, row schedule, build kernel) and ``Engine.i2i_topk``
(schedule, scoring kernel), after one warm-up call: median, min and max over ``--reps`` calls.  The scoring rate is
the bytes of S the kernel has to read, ``nnz(P) * n_items * 8``, over the scoring time, against 3.35 TB/s.

The reference's CooccurrenceModel (from oracle/_ref) is timed on the host: in full at the ML-1M shape; at the ML-20M
shape its build in full and its scoring on the first ``--ref-users-ml20m`` test users, scaled linearly to all test users
(an extrapolation, labelled so).  Prints one JSON line per shape.
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

SHAPES = {"ml1m": (6040, 3706, 1_000_000), "ml20m": (138_493, 26_744, 20_000_000)}
HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
        del out
    return dict(median_ms=float(np.median(ms)), min_ms=float(np.min(ms)), max_ms=float(np.max(ms)))


def reference_times(indptr, indices, values, shape, test_rows, ref_users):
    """the reference's build (in full) and get_recommendations on ``ref_users`` test users (None = all)."""
    from oracle import ref_driver as rd
    if rd.reference_root() is None:
        return None
    rd.import_reference()
    from polara.recommender.models import CooccurrenceModel
    n_users, n_items = shape
    user = np.repeat(np.arange(n_users, dtype=np.intp), np.diff(indptr))
    train = (np.c_[user, indices.astype(np.intp)], values.astype(np.float64))
    sub = test_rows if ref_users is None else test_rows[:ref_users]
    t_ptr = np.r_[0, np.cumsum(np.diff(indptr)[sub])]
    t_idx = np.concatenate([indices[indptr[u]:indptr[u + 1]] for u in sub])
    t_val = np.concatenate([values[indptr[u]:indptr[u + 1]] for u in sub])
    test = rd.csr_to_test_triplets(t_ptr, t_idx, t_val)

    class Data(rd.StubData):
        def get_test_shape(self, tensor_mode=False):
            return (len(sub), n_items)

    model = CooccurrenceModel(Data(shape, test=test, train=train))
    model.verbose = False
    model.verify_integrity = False
    t0 = time.perf_counter()
    model.build()
    t1 = time.perf_counter()
    model.get_recommendations()
    t2 = time.perf_counter()
    scale = len(test_rows) / len(sub)
    return dict(build_s=t1 - t0, score_s=(t2 - t1) * scale, score_users=len(sub),
                score_extrapolated=bool(scale != 1.0))


def run(name, reps, test_every, ref_users):
    import torch
    from polara_b200.engine import DeviceCSR, get_engine
    from polara_b200.synth import popularity_csr
    n_users, n_items, nnz = SHAPES[name]
    indptr, indices, values = popularity_csr(n_users, n_items, nnz, seed=3)
    eng = get_engine()
    a = eng.upload_csr(indptr, indices, values, (n_users, n_items))
    test_rows = np.arange(0, n_users, test_every)
    p_ptr = np.r_[0, np.cumsum(np.diff(indptr)[test_rows])].astype(np.int64)
    p_idx = np.concatenate([indices[indptr[u]:indptr[u + 1]] for u in test_rows])
    p_val = np.concatenate([values[indptr[u]:indptr[u + 1]] for u in test_rows])
    p = eng.upload_csr(p_ptr, p_idx, p_val, (len(test_rows), n_items))
    seen = (p.indptr, p.indices)
    build = timed(lambda: eng.cooc_build(a), reps)
    s = eng.cooc_build(a)
    score = timed(lambda: eng.i2i_topk(s, n_items, p, 10, seen=seen), reps)
    s_bytes = p.nnz * n_items * 8
    rec = dict(shape=name, users=n_users, items=n_items, train_nnz=int(a.nnz), test_users=len(test_rows),
               test_nnz=int(p.nnz), s_gb=n_items * s.shape[1] * 8 / 1e9, build=build, score=score,
               s_bytes_read=int(s_bytes), score_tb_per_s=s_bytes / (score["median_ms"] * 1e-3) / 1e12,
               hbm_fraction=s_bytes / (score["median_ms"] * 1e-3) / HBM_BYTES_PER_S, card=card())
    del s
    torch.cuda.empty_cache()
    if ref_users != 0:
        rec["reference"] = reference_times(indptr, indices, values, (n_users, n_items), test_rows,
                                           None if ref_users < 0 else ref_users)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="ml1m,ml20m")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--test-every", type=int, default=5)
    ap.add_argument("--ref-users-ml20m", type=int, default=300, help="0 skips the reference at the ML-20M shape")
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    lines = []
    for name in args.shapes.split(","):
        ref_users = 0 if args.no_reference else (-1 if name == "ml1m" else args.ref_users_ml20m)
        rec = run(name, args.reps, args.test_every, ref_users)
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

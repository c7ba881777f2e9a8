"""Sparse item-to-item matrix (pb200_cooc_build_csr, pb200_i2i_topk_csr) against the dense one, at the MovieLens-20M
shape where both fit, and at the BookCrossing shape where only the sparse one does.

    python scripts/i2i_sparse_bench.py [--shapes ml20m,bx] [--reps 3] [--ref-users 300] [--out FILE]

Synthetic data from ``polara_b200.synth.popularity_csr``.  The training matrix is every user; the test matrix is the
profile of every 5th user (20 % of the users).  Times are CUDA events around ``Engine.cooc_build_csr`` (transpose, both
passes, the host readback of the count between them) and ``Engine.i2i_topk_csr``, and around ``Engine.cooc_build`` /
``Engine.i2i_topk`` where the dense S fits: median, min and max over ``--reps`` calls after one warm-up.  The sparse and
dense lists are compared where both run.  The reference's CooccurrenceModel (from oracle/_ref) is timed on the host at
every shape: its build in full, its scoring on the first ``--ref-users`` test users scaled linearly to all of them (an
extrapolation, labelled so).  Prints one JSON line per shape.
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from i2i_bench import card, reference_times, timed  # noqa: E402

SHAPES = {"ml20m": (138_493, 26_744, 20_000_000), "bx": (278_858, 271_379, 1_150_000)}


def run(name, reps, ref_users):
    import torch
    from polara_b200.engine import cooc_csr_bytes, cooc_lds, get_engine
    from polara_b200.synth import popularity_csr
    n_users, n_items, nnz = SHAPES[name]
    indptr, indices, values = popularity_csr(n_users, n_items, nnz, seed=3)
    eng = get_engine()
    a = eng.upload_csr(indptr, indices, values, (n_users, n_items))
    test_rows = np.arange(0, n_users, 5)
    p_ptr = np.r_[0, np.cumsum(np.diff(indptr)[test_rows])].astype(np.int64)
    p_idx = np.concatenate([indices[indptr[u]:indptr[u + 1]] for u in test_rows])
    p_val = np.concatenate([values[indptr[u]:indptr[u + 1]] for u in test_rows])
    p = eng.upload_csr(p_ptr, p_idx, p_val, (len(test_rows), n_items))
    seen = (p.indptr, p.indices)
    dense_bytes = n_items * cooc_lds(n_items) * 8
    rec = dict(shape=name, users=n_users, items=n_items, train_nnz=int(a.nnz), test_users=len(test_rows),
               test_nnz=int(p.nnz), dense_s_bytes=dense_bytes, free_bytes=int(eng.free_bytes()), card=card())
    rec["sparse_build"] = timed(lambda: eng.cooc_build_csr(a), reps)
    s = eng.cooc_build_csr(a)
    rec["s_nnz"] = s.nnz
    rec["csr_bytes"] = cooc_csr_bytes(s.nnz, n_items)
    rec["sparse_score"] = timed(lambda: eng.i2i_topk_csr(s, p, 10, seen=seen), reps)
    got = [t.cpu().numpy() for t in eng.i2i_topk_csr(s, p, 10, seen=seen)]
    del s
    torch.cuda.empty_cache()
    if dense_bytes < eng.free_bytes() - (4 << 30):
        rec["dense_build"] = timed(lambda: eng.cooc_build(a), reps)
        sd = eng.cooc_build(a)
        rec["dense_score"] = timed(lambda: eng.i2i_topk(sd, n_items, p, 10, seen=seen), reps)
        want = [t.cpu().numpy() for t in eng.i2i_topk(sd, n_items, p, 10, seen=seen)]
        rec["lists_equal"] = all(x.tobytes() == y.tobytes() for x, y in zip(got, want))
        del sd
        torch.cuda.empty_cache()
    else:
        rec["dense_build"] = "does not fit: %d bytes for S" % dense_bytes
    if ref_users:
        rec["reference"] = reference_times(indptr, indices, values, (n_users, n_items), test_rows, ref_users)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="ml20m,bx")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-users", type=int, default=300, help="0 skips the reference")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    lines = []
    for name in args.shapes.split(","):
        rec = run(name, args.reps, args.ref_users)
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

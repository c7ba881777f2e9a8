"""HybridSVD build on the device: the matrix-free factored operator against forming ``K_u^T A K_i`` on the host.

    python scripts/hybrid_bench.py [--users 138493] [--items 26744] [--nnz 13900000] [--rank 50]
                                   [--item-fill 4] [--user-fill 2] [--ref-users 20000] [--out FILE]

A is synthetic (``polara_b200.synth.popularity_csr``) at the MovieLens-20M shape by default.  The Cholesky factors are
generated directly, with no factorisation: L is a random sparse lower-triangular matrix with a positive diagonal and
``--*-fill`` entries per row below it, and the permutation is random.  The script reports, for one build at ``--rank``:

* ``explicit``: the host time (scipy, float64) to form ``A K_i`` and then ``K_u^T (A K_i)``, plus the device build of
  that explicit operator (``B200SVDModel.build(operator=...)``, upload and transpose included);
* ``matrix_free``: the device build of ``B200HybridSVD`` on the same factors (``pb200_rsvd_factored``; K and K^T
  formed and uploaded, the projectors computed on the host, all included);
* ``nnz(A K_i) / nnz(A)`` and ``nnz(K_u^T A K_i) / nnz(A)``: the fill the explicit operator pays for;
* ``reference``: the reference's own matrix-free HybridSVD build (from oracle/_ref, ``svds`` on its ``LinearOperator``)
  on the first ``--ref-users`` users, all items, with the same factors restricted to them.

Times are wall-clock around calls that end in a device synchronise.  The card and its power limit are read in the same
run and printed with the result (one JSON line).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def random_factor(n, fill, seed):
    """``(L, perm)``: L lower-triangular CSR (float64) with a diagonal in [1, 2) and ~``fill`` entries per row at random
    columns below it (values ~ N(0, 0.3 / fill)); perm a random permutation."""
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(1, n, dtype=np.int64), fill)
    cols = (rng.random(rows.shape[0]) * rows).astype(np.int64)
    vals = rng.standard_normal(rows.shape[0]) * (0.3 / max(fill, 1))
    diag = np.arange(n, dtype=np.int64)
    low = sps.csr_matrix((np.r_[vals, 1.0 + rng.random(n)], (np.r_[rows, diag], np.r_[cols, diag])), shape=(n, n))
    low.sum_duplicates()
    low.sort_indices()
    return low, rng.permutation(n).astype(np.int64)


class _PairFactor:
    """the CHOLMOD-factor calls polara's CholeskyFactor makes, for a given ``(L, perm)``."""

    def __init__(self, low, perm):
        self._low, self._p = low.tocsc(), perm
        self._pinv = np.empty_like(perm)
        self._pinv[perm] = np.arange(perm.shape[0])

    def L(self):
        return self._low

    def P(self):
        return self._p

    def apply_P(self, b):
        return b[self._p]

    def apply_Pt(self, b):
        return b[self._pinv]

    def solve_Lt(self, b, use_LDLt_decomposition=False):
        from scipy.sparse.linalg import spsolve_triangular
        return spsolve_triangular(self._low.T.tocsr(), b, lower=False)


def sub_factor(low, perm, keep):
    """the user factor restricted to the first ``keep`` users, for timing the reference at a sub-size: the leading block
    of K = P^T L with the identity permutation.  It is not triangular, but the build only multiplies by a user factor
    (the triangular solve of the projectors is on the item side, which is kept whole)."""
    from polara_b200.models import cholesky_operator
    k = cholesky_operator(low, perm)[:keep, :keep].tocsr()
    return k, np.arange(keep, dtype=np.int64)


def reference_build(a, items, users, rank):
    """the reference's HybridSVD.build (matrix-free) on A with the given factors; returns seconds, or None."""
    from oracle import ref_driver as rd
    if rd.reference_root() is None:
        return None
    rd.import_reference()
    from polara.lib.cholesky import CholeskyFactor
    from polara.recommender.hybrid.models import HybridSVD
    coo = a.tocoo()
    data = rd.StubData(a.shape, train=(np.stack([coo.row, coo.col], axis=1).astype(np.intp), coo.data.astype(np.float64)))
    model = HybridSVD(data)
    model._sparse_mode = True
    model.verbose = False
    model.rank = rank
    model._cholesky = {data.fields.itemid: CholeskyFactor(_PairFactor(*items)),
                       data.fields.userid: None if users is None else CholeskyFactor(_PairFactor(*users))}
    t0 = time.perf_counter()
    model.build()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=138_493)
    ap.add_argument("--items", type=int, default=26_744)
    ap.add_argument("--nnz", type=int, default=13_900_000)
    ap.add_argument("--rank", type=int, default=50)
    ap.add_argument("--item-fill", type=int, default=4)
    ap.add_argument("--user-fill", type=int, default=2)
    ap.add_argument("--ref-users", type=int, default=20_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("hybrid_bench needs a CUDA device")
    from polara_b200.host import ArrayData
    from polara_b200.models import B200HybridSVD, B200SVDModel, cholesky_operator
    from polara_b200.synth import popularity_csr
    res = dict(card=card(), shape=[args.users, args.items], rank=args.rank, item_fill=args.item_fill,
               user_fill=args.user_fill)
    indptr, indices, values = popularity_csr(args.users, args.items, args.nnz, seed=3)
    a = sps.csr_matrix((values.astype(np.float64), indices, indptr), shape=(args.users, args.items))
    res["nnz_a"] = int(a.nnz)
    items = random_factor(args.items, args.item_fill, 4)
    users = random_factor(args.users, args.user_fill, 5) if args.user_fill > 0 else None
    coo = a.tocoo()
    data = ArrayData(np.stack([coo.row, coo.col], axis=1).astype(np.int64), coo.data, a.shape)

    # warm-up: one small factored build loads the modules and the allocator pool
    warm = B200HybridSVD(data)
    warm.verbose = False
    warm.rank = 4
    warm.item_cholesky_factor = items
    warm.build()
    torch.cuda.synchronize()

    t0 = time.perf_counter()
    model = B200HybridSVD(data)
    model.verbose = False
    model.rank = args.rank
    model.item_cholesky_factor, model.user_cholesky_factor = items, users
    model.build()
    torch.cuda.synchronize()
    res["matrix_free_s"] = time.perf_counter() - t0
    res["matrix_free_rsvd_s"] = model.last_timings["rsvd_s"]
    res["matrix_free_iters"] = model.last_timings["subspace_iters"]

    t0 = time.perf_counter()
    aki = (a @ cholesky_operator(*items)).tocsr()
    op = aki if users is None else (cholesky_operator(*users).T @ aki).tocsr()
    t1 = time.perf_counter()
    res["nnz_aki_over_a"] = aki.nnz / a.nnz
    res["nnz_op_over_a"] = op.nnz / a.nnz
    del aki
    plain = B200SVDModel(data)
    plain.verbose = False
    plain.rank = args.rank
    plain.build(operator=op)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    res["explicit_host_form_s"] = t1 - t0
    res["explicit_device_build_s"] = t2 - t1
    res["explicit_s"] = t2 - t0
    res["sigma_rel_diff"] = float(np.max(np.abs(plain.factors["singular_values"] - model.factors["singular_values"])
                                         / model.factors["singular_values"]))
    del op

    if args.ref_users > 0:
        m = min(args.ref_users, args.users)
        sub_users = None if users is None else sub_factor(users[0], users[1], m)
        t = reference_build(a[:m], items, sub_users, args.rank)
        res["reference"] = None if t is None else dict(users=m, items=args.items, seconds=t)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

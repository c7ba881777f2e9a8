"""Seeded synthetic interaction data (host side, numpy only).

Two generators:

* :func:`planted_ratings` -- small/medium problems with a planted low-rank
  preference structure and a geometrically decaying spectrum, so that the
  leading singular subspace is well separated (needed for a well-posed
  randomized-SVD vs ARPACK comparison, SURVEY.md §7.2).
* :func:`popularity_csr` -- large problems in CSR form directly (Zipf item
  popularity, log-normal user degrees, ratings 1..5 from a low-rank signal);
  used by ``bench.py`` for its workload shapes.
"""
from __future__ import annotations

import numpy as np


def planted_ratings(n_users, n_items, per_user, rank=8, decay=0.7, noise=0.25, seed=0,
                    levels=5):
    """Returns ``(user, item, rating)`` int64/int64/float64 arrays, no duplicate
    (user,item) pairs, users sorted ascending.  Every user gets ``per_user``
    distinct items (drawn with probability increasing in the planted affinity)."""
    rng = np.random.default_rng(seed)
    lam = decay ** np.arange(rank)
    x = rng.standard_normal((n_users, rank))
    y = rng.standard_normal((n_items, rank)) * lam
    pop = 1.0 / np.arange(1, n_items + 1) ** 0.5
    rng.shuffle(pop)
    aff = x @ y.T
    scale = aff.std()
    logits = np.log(pop)[None, :] + 1.5 * aff / scale
    gumbel = -np.log(-np.log(rng.random((n_users, n_items))))
    picked = np.argpartition(-(logits + gumbel), per_user - 1, axis=1)[:, :per_user]
    picked.sort(axis=1)
    user = np.repeat(np.arange(n_users, dtype=np.int64), per_user)
    item = picked.ravel().astype(np.int64)
    signal = aff[user, item] / scale + noise * rng.standard_normal(user.shape[0])
    # monotone map to 1..levels through empirical quantiles of the signal
    edges = np.quantile(signal, np.linspace(0, 1, levels + 1)[1:-1])
    rating = 1.0 + np.searchsorted(edges, signal).astype(np.float64)
    return user, item, rating


def popularity_csr(n_users, n_items, nnz_target, rank=16, seed=0, dtype=np.float32,
                   zipf=1.0, sigma_deg=1.0, chunk_users=200_000):
    """Large CSR ``(indptr int64, indices int32, data dtype)`` with sorted,
    duplicate-free column indices per row.  nnz ends up within a few percent of
    ``nnz_target`` (duplicates drawn for one user are dropped)."""
    rng = np.random.default_rng(seed)
    mean_deg = nnz_target / n_users
    deg = rng.lognormal(mean=0.0, sigma=sigma_deg, size=n_users)
    deg = np.clip(np.rint(deg * (mean_deg / deg.mean())), 1, max(1, n_items // 2)).astype(np.int64)
    w = 1.0 / np.arange(1, n_items + 1, dtype=np.float64) ** zipf
    cdf = np.cumsum(w)
    cdf /= cdf[-1]
    perm = rng.permutation(n_items).astype(np.int32)   # decouple id from popularity rank
    lam = (0.85 ** np.arange(rank)).astype(np.float32)
    yf = (rng.standard_normal((n_items, rank)).astype(np.float32)) * lam
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    idx_parts, val_parts = [], []
    for lo in range(0, n_users, chunk_users):
        hi = min(lo + chunk_users, n_users)
        d = deg[lo:hi]
        rows = np.repeat(np.arange(hi - lo, dtype=np.int64), d)
        cols = perm[np.searchsorted(cdf, rng.random(rows.shape[0]))]
        key = rows * n_items + cols
        key = np.unique(key)                       # sorts by (row, col), drops duplicates
        rows = key // n_items
        cols = (key - rows * n_items).astype(np.int32)
        xf = rng.standard_normal((hi - lo, rank)).astype(np.float32)
        sig = np.einsum("ij,ij->i", xf[rows], yf[cols])
        sig += 0.3 * rng.standard_normal(sig.shape[0]).astype(np.float32)
        rating = np.clip(np.rint(3.0 + 1.2 * sig / max(1e-6, sig.std())), 1, 5).astype(dtype)
        counts = np.bincount(rows, minlength=hi - lo)
        indptr[lo + 1:hi + 1] = counts
        idx_parts.append(cols)
        val_parts.append(rating)
    np.cumsum(indptr, out=indptr)
    return indptr, np.concatenate(idx_parts), np.concatenate(val_parts)

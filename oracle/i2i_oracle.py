"""f64 numpy/scipy restatement of the reference's item-to-item model (CooccurrenceModel, polara/recommender/models.py:
693-725) -- TEST INFRASTRUCTURE.  Ties, which the reference leaves to argpartition / quicksort, are broken by the lower
item id here; everything else follows the cited lines."""
import sys

import numpy as np
import scipy.sparse as sps

from oracle.polara_oracle import _user_slices


def cooc_matrix(train_idx, train_val, shape, implicit=False):
    """build(), models.py:696-709: A = get_training_matrix() (coo -> csr sums duplicates, :169-172), sign with
    ``implicit``, S = A^T A, setdiag(0), eliminate_zeros().  Returns S as an f64 CSR."""
    idx = np.asarray(train_idx)
    a = sps.coo_matrix((np.asarray(train_val, dtype=np.float64), (idx[:, 0], idx[:, 1])), shape=tuple(shape[:2])).tocsr()
    if implicit:
        a.data = np.sign(a.data)
    s = (a.T @ a).tocsr()
    s.setdiag(0)
    s.eliminate_zeros()
    return s


def test_matrix(user, item, fdbk, shape, implicit=False):
    """get_test_matrix (models.py:180-211) -- zero feedback dropped, duplicates summed -- and the sign of
    slice_recommendations with ``implicit`` (:716-717)."""
    fdbk = np.asarray(fdbk, dtype=np.float64)
    keep = fdbk != 0
    p = sps.csr_matrix((fdbk[keep], (np.asarray(user)[keep], np.asarray(item)[keep])), shape=tuple(shape[:2]))
    if implicit:
        p.data = np.sign(p.data)
    return p


def scores(p, s):
    """the score block P S (lib/sparse.py:45-47) as an f64 CSR holding the nonzero sums only, as csr_matmat stores them."""
    out = (p @ s).tocsr()
    out.eliminate_zeros()
    return out


def nnz_max(memory_hard_limit):
    """get_nnz_max, lib/sparse.py:15-22."""
    per_entry = sys.getsizeof(()) + 2 * (sys.getsizeof(1.0) + np.dtype(np.intp).itemsize)
    return int(memory_hard_limit * (1024 ** 3) / per_entry)


def chunk_modes(nnz_u, n_items, topk, memory_hard_limit, dense_output=False):
    """per chunk ``(start, stop, dense)``: the chunks of _get_slices_idx (models.py:215-225, utils.py:7-53; the limit is
    ``memory_hard_limit`` because get_available_memory's bytes are read as GB) and sparse_dot's choice (lib/sparse.py:
    25-55): dense with dense_output, above get_nnz_max, or above half the block (check_sparsity)."""
    nnz_u = np.asarray(nnz_u)
    slices = _user_slices((len(nnz_u), int(n_items)), topk, 1, memory_hard_limit or None, None)
    out = []
    for a, b in slices:
        nnz = int(nnz_u[a:b].sum())
        out.append((int(a), int(b), bool(dense_output or nnz > nnz_max(memory_hard_limit)
                                         or nnz > 0.5 * (b - a) * int(n_items))))
    return out


def _order(score, ids):
    """ids by (score desc, id asc)."""
    return ids[np.lexsort((ids, -score))]


def dense_rule(row, seen, k, filter_seen=True):
    """toarray + downvote_seen_items + topsort (models.py:510-519, 561-563, 488-491): unseen items by (score desc,
    id asc), zero scores included, then the seen ones in the same order; every item in that order without filtering."""
    row = np.asarray(row, dtype=np.float64)
    ids = np.arange(len(row))
    if not filter_seen:
        return _order(row, ids)[:k]
    is_seen = np.zeros(len(row), dtype=bool)
    is_seen[np.asarray(seen, dtype=np.int64)] = True
    return np.r_[_order(row[~is_seen], ids[~is_seen]), _order(row[is_seen], ids[is_seen])][:k]


def sparse_rule(cols, vals, k):
    """topscore (models.py:524-560): the nonzero scores by (score desc, id asc), then -1 (_pad_const, :73) up to k.
    Seen items stay, filter_seen or not: downvote_seen_items' sparse branch (models.py:501-509) ends in
    ``recs -= seen_recs``, and scipy's sparse matrices have no in-place subtraction, so Python rebinds the local name to
    a new matrix and the caller's score block keeps the seen scores."""
    cols = np.asarray(cols, dtype=np.int64)
    vals = np.asarray(vals, dtype=np.float64)
    keep = vals != 0
    top = _order(vals[keep], cols[keep])[:k]
    return np.r_[top, -np.ones(k - len(top), dtype=np.int64)]


def recommend(train_idx, train_val, train_shape, test_user, test_item, test_fdbk, test_shape, topk=10,
              filter_seen=True, implicit=False, dense_output=False, memory_hard_limit=1):
    """get_recommendations (models.py:391-405, 359-371) of CooccurrenceModel.  Returns ``(lists int64 [m x topk],
    modes [(start, stop, dense)], nnz_u, scores f64 CSR)``."""
    s = cooc_matrix(train_idx, train_val, train_shape, implicit)
    p = test_matrix(test_user, test_item, test_fdbk, test_shape, implicit)
    sc = scores(p, s)
    nnz_u = np.diff(sc.indptr)
    seen = sps.csr_matrix((np.ones(len(test_user)), (np.asarray(test_user), np.asarray(test_item))),
                          shape=tuple(test_shape[:2]))
    modes = chunk_modes(nnz_u, test_shape[1], topk, memory_hard_limit, dense_output)
    out = np.empty((test_shape[0], topk), dtype=np.int64)
    for a, b, dense in modes:
        for u in range(a, b):
            sn = seen.indices[seen.indptr[u]:seen.indptr[u + 1]]
            lo, hi = sc.indptr[u], sc.indptr[u + 1]
            if dense:
                row = np.zeros(test_shape[1])
                row[sc.indices[lo:hi]] = sc.data[lo:hi]
                out[u] = dense_rule(row, sn, topk, filter_seen)
            else:
                out[u] = sparse_rule(sc.indices[lo:hi], sc.data[lo:hi], topk)
    return out, modes, nnz_u, sc

"""f64 numpy/scipy restatement of the reference's SimilarityAggregation (polara/recommender/hybrid/models.py:25-44) --
TEST INFRASTRUCTURE.  Scores are ``sparse_dot(P, S)``: ``P S^T`` (lib/sparse.py:48), or with ``dense_output`` what
``csc_matvec`` makes of the stored arrays of S (lib/sparse.py:40-43, 119-130): ``P S`` for relations held as CSR.  The
lists then follow the item-to-item model's chunk rules (oracle/i2i_oracle.py)."""
import numpy as np
import scipy.sparse as sps

from oracle import i2i_oracle as io


def similarity_matrix(relations):
    """build(), hybrid/models.py:33-37: a copy of the relations with a zero diagonal and no stored zeros."""
    s = relations.copy()
    s.setdiag(0)
    s.eliminate_zeros()
    return s


def scoring_operand(s, dense_output=False):
    """the matrix M with scores = P M: S^T, or S for ``dense_output`` on CSR relations (csc_matvec reads them as CSC)."""
    m = s if (dense_output and s.format == "csr") else s.T
    return sps.csr_matrix(m, dtype=np.float64)


def test_matrix(user, item, fdbk, shape, implicit=False):
    """get_test_matrix (models.py:180-211), then ones for every stored value with ``implicit`` (hybrid/models.py:41-42)."""
    p = io.test_matrix(user, item, fdbk, shape)
    if implicit:
        p.data = np.ones_like(p.data)
    return p


def recommend(relations, test_user, test_item, test_fdbk, test_shape, topk=10, filter_seen=True, implicit=False,
              dense_output=False, memory_hard_limit=1):
    """get_recommendations of SimilarityAggregation.  Returns ``(lists int64 [m x topk], modes, nnz_u, scores f64 CSR)``."""
    s = similarity_matrix(relations)
    p = test_matrix(test_user, test_item, test_fdbk, test_shape, implicit)
    sc = io.scores(p, scoring_operand(s, dense_output))
    nnz_u = np.diff(sc.indptr)
    seen = sps.csr_matrix((np.ones(len(test_user)), (np.asarray(test_user), np.asarray(test_item))),
                          shape=tuple(test_shape[:2]))
    modes = io.chunk_modes(nnz_u, test_shape[1], topk, memory_hard_limit, dense_output)
    out = np.empty((test_shape[0], topk), dtype=np.int64)
    for a, b, dense in modes:
        for u in range(a, b):
            sn = seen.indices[seen.indptr[u]:seen.indptr[u + 1]]
            lo, hi = sc.indptr[u], sc.indptr[u + 1]
            if dense:
                row = np.zeros(test_shape[1])
                row[sc.indices[lo:hi]] = sc.data[lo:hi]
                out[u] = io.dense_rule(row, sn, topk, filter_seen)
            else:
                out[u] = io.sparse_rule(sc.indices[lo:hi], sc.data[lo:hi], topk)
    return out, modes, nnz_u, sc

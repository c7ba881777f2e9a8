"""f64 restatement of HybridSVD (polara/recommender/hybrid/models.py:335-394) for the recorded cases of
``tests/golden/hybrid_cases.npz``  --  TEST INFRASTRUCTURE.

Factors come from :mod:`oracle.cholmod_stub` (the stand-in the fixture was recorded with), the operator
``K_u^T A K_i`` is formed explicitly in float64 and factorised by ``svds``, and scores are
``P . (K v) . (K^-T v)^T`` with the reference's seen-item handling and top-k order.
"""
import numpy as np
import scipy.linalg
import scipy.sparse as sps

from oracle import cholmod_stub
from oracle import polara_oracle as po


def case(g, name):
    """the ``<name>_*`` arrays of a fixture dict, without the prefix."""
    p = name + "_"
    return {k[len(p):]: v for k, v in g.items() if k.startswith(p)}


def beta(features_weight):
    """hybrid/models.py:292-293."""
    return (1.0 - features_weight) / features_weight


def similarity(c, side):
    """the recorded similarity matrix of ``side`` ('item' / 'user') as a float64 CSR, or None."""
    if not bool(c[side + "_present"]):
        return None
    n = len(c[side + "_sim_indptr"]) - 1
    return sps.csr_matrix((c[side + "_sim_data"], c[side + "_sim_indices"], c[side + "_sim_indptr"]), shape=(n, n))


def factor(c, side):
    """the stub's CHOLMOD factor of ``S + beta I`` for ``side``, or None."""
    s = similarity(c, side)
    return None if s is None else cholmod_stub.cholesky(s, beta=beta(float(c["features_weight"])))


def k_matrix(f):
    """K = P^T L as a dense float64 matrix (``K v = apply_Pt(L v)``)."""
    low = f.L().toarray()
    return f.apply_Pt(low)


def training_matrix(c):
    """get_training_matrix(dtype=float64) (models.py:160-177), rescaled for the scaled variant (models.py:891-895)."""
    idx = c["train_idx"]
    a = sps.csr_matrix((c["train_val"].astype(np.float64), (idx[:, 0], idx[:, 1])), shape=tuple(c["train_shape"]))
    if bool(c["scaled"]):
        a = po.scaled_training_matrix(a, float(c["row_scaling"]), float(c["col_scaling"]))
    return a


def operator(a, k_items=None, k_users=None):
    """the explicit ``K_u^T A K_i`` (dense float64); a None factor is the identity."""
    op = a.toarray() if sps.issparse(a) else np.asarray(a, dtype=np.float64)
    if k_items is not None:
        op = op @ k_items
    if k_users is not None:
        op = k_users.T @ op
    return op


def projectors(f, v):
    """build_item_projector (hybrid/models.py:315-326): ``(K^-T v, K v)``."""
    low = f.L().toarray()
    left = f.apply_Pt(scipy.linalg.solve_triangular(low.T, v, lower=False))
    right = f.apply_Pt(low @ v)
    return left, right


def recommend(c, vl, vr, topk=10):
    """the reference's lists for projectors ``vl`` / ``vr`` (slice_recommendations, hybrid/models.py:390-394, then
    downvote_seen_items and get_topk_elements); one chunk at these sizes."""
    shape = tuple(c["test_shape"])
    p = po._test_matrix(c["test_user"], c["test_item"], c["test_fdbk"], shape[0], shape[1])
    scores = po.hybrid_slice_scores(p, vl, vr)
    po.downvote_seen_items(scores, c["test_user"], c["test_item"])
    return po.get_topk_elements(scores, topk), scores

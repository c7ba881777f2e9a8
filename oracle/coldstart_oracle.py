"""f64 restatement of the item cold-start SVD models (polara/recommender/coldstart/models.py:149-257) for the recorded
cases of ``tests/golden/coldstart_cases.npz``  --  TEST INFRASTRUCTURE.

From recorded factors: the feature mapping ``W = F^T V`` (or ``F^T V_r`` with HybridSVD's right projector), its
transform ``pinv(W^T W)``, the scores ``(F_cold W) pinv(W^T W) (U diag s)^T`` of every (cold item, user) pair and
their top-k users per cold item under the reference's order (nothing is seen in cold start; ties by the lower user id).
"""
import numpy as np
import scipy.sparse as sps

from oracle import polara_oracle as po
from oracle.hybrid_oracle import case  # noqa: F401  (the ``<name>_*`` arrays of a fixture dict)


def csr(c, key):
    """the recorded CSR ``<key>_{indptr,indices,data,shape}`` as a float64 scipy CSR."""
    return sps.csr_matrix((c[key + "_data"], c[key + "_indices"], c[key + "_indptr"]), shape=tuple(c[key + "_shape"]))


def mapping_source(c):
    """what W is built from: the item factors, or HybridSVD's right item projector (:233-236, 247-251)."""
    return c["projector_right"] if bool(c["hybrid"]) else c["item_factors"]


def feature_mapping(f, v):
    """compute_item_features_mapping (:233-236, 247-251): ``W = F^T v``."""
    return np.asarray(f.T.dot(np.asarray(v, dtype=np.float64)))


def transform(w):
    """update_item_features_transform (:192-195): ``pinv(W^T W)``."""
    return np.linalg.pinv(w.T @ w)


def scores(f_cold, w, t, u, s):
    """slice_recommendations (:209-222), float64: ``[n_cold x n_users]``."""
    r = u.shape[1]
    w, t = np.asarray(w)[:, :r], np.asarray(t)[:r, :r]
    return (np.asarray(f_cold @ w) @ t) @ (np.asarray(u) * np.asarray(s)[None, :r]).T


def recommend(f_cold, w, t, u, s, topk):
    """top-k users per cold item (get_topk_elements, models.py:522-564, filter_seen off) and the scores."""
    sc = scores(f_cold, w, t, u, s)
    return po.get_topk_elements(sc, topk), sc


def truncated(c, rank):
    """the recorded factors cut to ``rank`` (SVDModel._check_reduced_rank, models.py:819-832) and the transform
    recomputed there (:169-183): ``(u, s, w, t)``."""
    w = c["W"][:, :rank]
    return c["user_factors"][:, :rank], c["singular_values"][:rank], w, transform(w)


def data(c, **kwargs):
    """the case's :class:`polara_b200.host.ColdStartData` (holdout, F and F_cold as recorded; nothing left to drop)."""
    from polara_b200.host import ColdStartData
    f_cold_rows = np.zeros((int(c["cold_new"].max()) + 1, c["F_shape"][1]))
    fc = csr(c, "F_cold").toarray()
    f_cold_rows[c["cold_new"]] = fc
    return ColdStartData(c["train_idx"], c["train_val"], c["train_shape"], c["holdout_cold"], c["holdout_user"],
                         c["holdout_fdbk"], csr(c, "F"), sps.csr_matrix(f_cold_rows), n_users=int(c["n_users"]),
                         representative_users=c["repr_users"] if len(c["repr_users"]) else None, **kwargs)

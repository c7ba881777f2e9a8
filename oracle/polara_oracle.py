"""CPU oracle for the Polara hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import this module.  The product path
(``polara_b200``) never imports it and has no CPU fallback.

This is a numpy/scipy *restatement* (written from the algorithm, not copied) of
the reference functions that SURVEY.md §8(a) lists.  Every function cites the
reference lines it follows (paths relative to the reference checkout).

Third-party arithmetic the reference itself delegates to and that is NOT under
the reference tree: ``scipy.sparse.linalg.svds`` (ARPACK; reference pin
``scipy>=0.16.0`` in conda_req.txt:11, installed here: scipy 1.18.1).  The
oracle calls the same routine at the same call sites (models.py:844,
lib/tensor.py:71,75,79) because that *is* the reference's algorithm.

Pinning: the reference's own tests hold no vector for this path (SURVEY.md §4).
The oracle is therefore pinned against outputs of the reference itself, recorded
by ``oracle/make_golden.py`` and committed under
``tests/golden/`` (see tests/test_oracle_golden.py, tests/test_oracle_vs_reference.py).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sps
from scipy.sparse.linalg import svds

__all__ = [
    "topsort", "get_topk_elements", "downvote_seen_items", "svd_build",
    "svd_slice_scores", "rescale_matrix", "scaled_training_matrix",
    "get_chunk_size", "range_division", "recommend_svd", "ttm3d", "hooi",
    "flatten_scores", "coffee_slice_scores", "recommend_coffee",
    "rank_key_order",
]


# ----------------------------------------------------------------------------
# top-k and seen-item masking
# ----------------------------------------------------------------------------
def topsort(a, topk):
    """models.py:488-491 -- ids of the ``topk`` largest entries of 1-d ``a``,
    ordered by descending value (introselect partition, then sort of the part)."""
    a = np.asarray(a)
    part = np.argpartition(a, -topk)[-topk:]
    order = np.argsort(-a[part])
    return part[order]


def get_topk_elements(scores, topk):
    """models.py:561-563 (dense branch) -- row-wise ``topsort``."""
    scores = np.asarray(scores)
    out = np.empty((scores.shape[0], topk), dtype=np.intp)
    for i in range(scores.shape[0]):
        out[i] = topsort(scores[i], topk)
    return out


def downvote_seen_items(scores, seen_rows, seen_cols):
    """models.py:510-519 (dense branch) -- in place.

    Seen entries are pushed below the block minimum while keeping their mutual
    order: ``new = min(S) - (max(S_seen) - S_seen) - 1``."""
    if len(seen_rows) == 0:
        # reference: ``seen_data.max()`` of an empty selection raises ValueError
        raise ValueError("zero-size array to reduction operation maximum")
    flat = np.ravel_multi_index((np.asarray(seen_rows), np.asarray(seen_cols)), scores.shape)
    seen_vals = scores.flat[flat]
    scores.flat[flat] = scores.min() - (seen_vals.max() - seen_vals) - 1
    return scores


def rank_key_order(scores_row, seen_cols_row, topk):
    """Order-equivalent statement of downvote+topsort for ONE row, free of the
    block-global min/max: unseen items by descending score, then seen items by
    descending score (what models.py:517-519 achieves).  Ties are broken by the
    lower item id (the reference leaves tie order unspecified, models.py:488-491).
    Used by tests to state the contract the CUDA path implements."""
    s = np.asarray(scores_row, dtype=np.float64)
    seen = np.zeros(s.shape[0], dtype=bool)
    seen[np.asarray(seen_cols_row, dtype=np.intp)] = True
    order = np.lexsort((np.arange(s.shape[0]), -s, seen))
    return order[:topk]


# ----------------------------------------------------------------------------
# PureSVD build + folding-in scores
# ----------------------------------------------------------------------------
def svd_build(matrix, rank, return_u=False):
    """models.py:835-855 -- ``svds(A, k=rank)`` (ARPACK, ascending) flipped to
    descending.  Returns ``(V [n_items x rank], sigma [rank], U or None)``."""
    a = sps.csr_matrix(matrix, dtype=np.float64)
    mode = True if return_u else "vh"
    u, s, vt = svds(a, k=rank, return_singular_vectors=mode)
    v = np.ascontiguousarray(vt[::-1, :]).T
    s = np.ascontiguousarray(s[::-1])
    if u is not None and return_u:
        u = np.ascontiguousarray(u[:, ::-1])
    else:
        u = None
    return v, s, u


def svd_slice_scores(test_matrix, v):
    """models.py:857-861 -- folding-in scores ``(P V) V^T`` (dense f64)."""
    return np.asarray(test_matrix.dot(v)).dot(v.T)


def hybrid_item_projectors(cholesky_items, v):
    """hybrid/models.py:315-325 (``build_item_projector``): left = ``L^-T v`` (``cholesky_items.T.solve(v)``),
    right = ``L v`` (``cholesky_items.dot(v)``) for the Cholesky factor ``L`` (dense lower-triangular here; CHOLMOD's sparse
    factor in the reference) of the item similarity matrix."""
    from scipy.linalg import solve_triangular
    chol = np.asarray(cholesky_items, dtype=np.float64)
    return solve_triangular(chol.T, v, lower=False), chol @ v


def hybrid_slice_scores(test_matrix, vl, vr):
    """hybrid/models.py:390-394 -- ``HybridSVD.slice_recommendations``: ``scores = P . vr . vl^T`` (dense f64)."""
    return np.asarray(test_matrix.dot(vr)).dot(vl.T)


def rescale_matrix(matrix, scaling, axis):
    """preprocessing/matrices.py:71-93 with ``binary=True`` (the default used
    by ScaledMatrixMixin): scale rows (axis=1) or columns (axis=0) by
    ``sqrt(count)**(scaling-1)``, ``count`` the line's stored entries
    (``getnnz``: explicit zeros included); zero-count lines keep an
    (irrelevant) factor.

    There is no early return at ``scaling == 1``: the reference forms the
    product with ``diags(...)`` then too, and a scipy sparse product stores
    only nonzero results.  So the result never holds an explicit zero, and in
    ``scaled_training_matrix`` the column counts, taken after the row pass,
    exclude the zeros that the row counts include."""
    m = sps.csr_matrix(matrix, dtype=np.float64)
    counts = np.asarray(m.getnnz(axis=axis)).ravel()
    norm = np.sqrt(counts)
    factor = np.ones_like(norm)
    nz = norm != 0
    factor[nz] = np.power(norm[nz], scaling - 1)
    d = sps.diags(factor)
    out = (m @ d).tocsr() if axis == 0 else (d @ m).tocsr()
    out.eliminate_zeros()          # what the sparse product does; stated here rather than left to scipy
    return out


def scaled_training_matrix(matrix, row_scaling=1, col_scaling=0.4):
    """models.py:891-895 -- rows first (axis=1), then columns (axis=0)."""
    m = rescale_matrix(matrix, row_scaling, 1)
    return rescale_matrix(m, col_scaling, 0)


# ----------------------------------------------------------------------------
# user chunking (defines the CPU granularity only)
# ----------------------------------------------------------------------------
def range_division(length, fit_size):
    """utils.py:7-13."""
    n_chunks = length // fit_size + int(length % fit_size > 0)
    base, rem = divmod(length, n_chunks)
    sizes = [0] + rem * [base + 1] + (n_chunks - rem) * [base]
    return np.cumsum(sizes)


def get_chunk_size(shape, result_width, scores_multiplier=1, memory_hard_limit=1.0,
                   available_gb=None):
    """utils.py:16-47 with int64 results / float64 scores.  ``available_gb`` is
    the free host memory in GiB (the reference reads psutil); None = unlimited."""
    chunk = shape[0]
    s0, s1 = shape[0] / 1024.0, shape[1] / 1024.0
    item_kb = 8 / 1024.0
    result_mem = s0 * (result_width / 1024.0) * item_kb
    scores_mem = s0 * s1 * scores_multiplier * item_kb
    limit = np.inf if available_gb is None else 0.8 * available_gb
    if memory_hard_limit:
        limit = min(limit, memory_hard_limit)
    if scores_mem + result_mem > limit:
        chunk = min(int((limit - result_mem)
                        / (s1 * item_kb * (scores_multiplier / 1024.0) + item_kb / 1024.0 ** 2) - 1),
                    chunk)
        if chunk <= 0:
            raise MemoryError()
    return chunk


def _user_slices(shape, topk, scores_multiplier, memory_hard_limit, available_gb):
    chunk = get_chunk_size(shape, topk, scores_multiplier, memory_hard_limit, available_gb)
    bounds = range_division(shape[0], chunk)
    return list(zip(bounds[:-1], bounds[1:]))


def _slice_coo(user, item, fdbk, start, stop):
    """models.py:260-270."""
    sel = (user >= start) & (user < stop)
    return user[sel] - start, item[sel], fdbk[sel]


def _test_matrix(user, item, fdbk, n_users, n_items):
    """models.py:180-211 -- zero feedback is dropped from P but the unfiltered
    triplets remain the seen list."""
    keep = fdbk != 0
    return sps.csr_matrix((fdbk[keep].astype(np.float64), (user[keep], item[keep])),
                          shape=(n_users, n_items))


def recommend_svd(test_user, test_item, test_fdbk, shape, v, topk=10, filter_seen=True,
                  memory_hard_limit=1.0, available_gb=None, user_range=None):
    """models.py:359-405 + 857-861 -- the sequential chunk driver for SVDModel.

    ``test_*`` are the user-sorted COO arrays of ``_get_test_data`` (users
    re-based to 0..m-1).  ``user_range=(a,b)`` restricts the work to those
    users (used for bounded CPU-baseline samples); chunk boundaries are still
    the reference's.  Returns int64 ``[m x topk]``."""
    test_user = np.asarray(test_user)
    test_item = np.asarray(test_item)
    test_fdbk = np.asarray(test_fdbk)
    slices = _user_slices(shape, topk, 1, memory_hard_limit, available_gb)
    if user_range is not None:
        slices = [(a, b) for (a, b) in slices if a >= user_range[0] and b <= user_range[1]]
        base = slices[0][0]
        out = np.empty((slices[-1][1] - base, topk), dtype=np.int64)
    else:
        base = 0
        out = np.empty((shape[0], topk), dtype=np.int64)
    for start, stop in slices:
        stop = min(stop, shape[0])
        u, i, f = _slice_coo(test_user, test_item, test_fdbk, start, stop)
        p = _test_matrix(u, i, f, stop - start, shape[1])
        scores = svd_slice_scores(p, v)
        if filter_seen:
            downvote_seen_items(scores, u, i)
        out[start - base:stop - base] = get_topk_elements(scores, topk)
    return out


# ----------------------------------------------------------------------------
# CoFFee: HOOI build and scoring
# ----------------------------------------------------------------------------
def ttm3d(idx, val, shape, u, v, mode0, mode1, mode2):
    """lib/tensor.py:7-19 + lib/sparse.py:203-216 (dttm_seq) --
    ``res[i0,:,:] += val * u[i1,:] (x) v[i2,:]`` over all nnz;
    result ``[shape[mode0], u.shape[1], v.shape[1]]``."""
    idx = np.asarray(idx)
    n0, r1, r2 = shape[mode0], u.shape[1], v.shape[1]
    res = np.zeros((n0, r1 * r2))
    step = max(1, (1 << 24) // max(1, r1 * r2))
    for lo in range(0, len(val), step):
        hi = min(lo + step, len(val))
        kr = (u[idx[lo:hi, mode1], :, None] * v[idx[lo:hi, mode2], None, :]).reshape(hi - lo, -1)
        kr *= np.asarray(val[lo:hi])[:, None]
        sel = sps.csr_matrix((np.ones(hi - lo), (idx[lo:hi, mode0], np.arange(hi - lo))),
                             shape=(n0, hi - lo))
        res += sel @ kr
    return res.reshape(n0, r1, r2)


def hooi(idx, val, shape, core_shape, num_iters=25, growth_tol=0.01, seed=None,
         init=None, return_trace=False):
    """lib/tensor.py:37-96 -- HOOI / Tucker-ALS on a COO 3-way tensor.

    ``init=(u1, u2)`` overrides the random start (lib/tensor.py:57-63) so that a
    device run can be started from identical factors.  Returns
    ``(u0, u1, u2, core)`` (+ the list of core norms when ``return_trace``)."""
    r0, r1, r2 = core_shape
    if init is None:
        rs = np.random if seed is None else np.random.RandomState(seed)
        u1 = np.linalg.qr(rs.rand(shape[1], r1), mode="reduced")[0]
        u2 = np.linalg.qr(rs.rand(shape[2], r2), mode="reduced")[0]
    else:
        u1, u2 = (np.array(x, dtype=np.float64) for x in init)
    norm_old = 0.0
    trace = []
    for _ in range(num_iters):
        unf = ttm3d(idx, val, shape, u2, u1, 0, 2, 1).reshape(shape[0], r1 * r2)
        uu, ss, _ = svds(unf, k=r0, return_singular_vectors="u")
        u0 = np.ascontiguousarray(uu[:, ::-1])

        unf = ttm3d(idx, val, shape, u2, u0, 1, 2, 0).reshape(shape[1], r0 * r2)
        uu, ss, _ = svds(unf, k=r1, return_singular_vectors="u")
        u1 = np.ascontiguousarray(uu[:, ::-1])

        unf = ttm3d(idx, val, shape, u1, u0, 2, 1, 0).reshape(shape[2], r0 * r1)
        uu, ss, vv = svds(unf, k=r2, return_singular_vectors=True)
        u2 = np.ascontiguousarray(uu[:, ::-1])

        norm_new = np.linalg.norm(ss)
        trace.append(norm_new)
        growth = (norm_new - norm_old) / norm_new
        norm_old = norm_new
        if growth < growth_tol:
            break
    core = np.ascontiguousarray((ss[:, None] * vv)[::-1, :]).reshape(r2, r1, r0).transpose(2, 1, 0)
    if return_trace:
        return u0, u1, u2, core, trace
    return u0, u1, u2, core


def round_core(core, mode, rank):
    """models.py:966-980 -- truncated SVD of the mode-``mode`` unfolding of a Tucker core (the
    remaining modes flattened in Fortran order); returns the rotation ``[r_mode x rank]`` to apply
    to that mode's factor and the shrunken core (same mode order as the input)."""
    order = [mode] + [d for d in range(core.ndim) if d != mode]
    rest = [core.shape[d] for d in order[1:]]
    unfolded = np.reshape(np.transpose(core, order), (core.shape[mode], -1), order="F")
    u, s, vt = np.linalg.svd(unfolded, full_matrices=False)
    folded = np.reshape(np.ascontiguousarray(s[:rank, None] * vt[:rank]), [rank] + rest, order="F")
    return u[:, :rank], np.transpose(folded, np.argsort(order))


def reduce_tucker_rank(factors, core, mlrank):
    """models.py:949-963 -- CoffeeModel._check_reduced_rank: for every mode whose factor is wider
    than the requested rank, rotate the factor and shrink the core; ``None`` if any factor is
    narrower (the model must be rebuilt)."""
    factors = list(factors)
    for mode, rank in enumerate(mlrank):
        if factors[mode].shape[1] < rank:
            return None
        if factors[mode].shape[1] > rank:
            rot, core = round_core(core, mode, rank)
            factors[mode] = factors[mode].dot(rot)
    return factors, core


def flatten_scores(tensor_scores, flattener=None):
    """models.py:983-1006 -- collapse the trailing feedback axis."""
    flattener = slice(None) if flattener is None else flattener
    if isinstance(flattener, str):
        return getattr(np, flattener)(tensor_scores, axis=-1)
    if isinstance(flattener, int):
        return tensor_scores[..., flattener]
    if isinstance(flattener, (list, slice)):
        return np.sum(tensor_scores[..., flattener], axis=-1)
    if isinstance(flattener, tuple):
        sl, how = flattener
        return getattr(np, how)(tensor_scores[..., sl or slice(None)], axis=-1)
    if callable(flattener):
        return flattener(tensor_scores)
    raise ValueError("Unrecognized value for flattener attribute")


def coffee_slice_scores(user, item, fdbk_idx, n_users, v, w, flattener=None):
    """models.py:1042-1054 + lib/sparse.py:190-200 -- per-nnz outer products
    ``v[i,:] (x) w[f,:]``, summed per user, contracted with ``flatten(w^T)``,
    then ``. V^T``.  ``user`` must be sorted (re-based to 0..n_users-1)."""
    user = np.asarray(user)
    outer = v[np.asarray(item), :, None] * w[np.asarray(fdbk_idx), None, :]
    starts = np.r_[0, np.where(np.diff(user))[0] + 1]
    per_user = np.add.reduceat(outer, starts)
    # reduceat yields one row per *present* user; the reference relies on every
    # user of the slice being present (models.py:1050).
    assert per_user.shape[0] == n_users
    wt_flat = flatten_scores(w.T, flattener)
    return np.tensordot(per_user, wt_flat, axes=(2, 0)).dot(v.T)


def recommend_coffee(test_user, test_item, test_fdbk_idx, shape, v, w, topk=10,
                     flattener=None, filter_seen=True, memory_hard_limit=1.0,
                     available_gb=None):
    """models.py:359-405 + 1042-1054 -- chunk driver for CoffeeModel
    (``scores_multiplier`` = r2, models.py:216-221)."""
    test_user = np.asarray(test_user)
    test_item = np.asarray(test_item)
    test_fdbk_idx = np.asarray(test_fdbk_idx)
    out = np.empty((shape[0], topk), dtype=np.int64)
    for start, stop in _user_slices(shape, topk, w.shape[1], memory_hard_limit, available_gb):
        u, i, f = _slice_coo(test_user, test_item, test_fdbk_idx, start, stop)
        scores = coffee_slice_scores(u, i, f, stop - start, v, w, flattener)
        if filter_seen:
            downvote_seen_items(scores, u, i)
        out[start:stop] = get_topk_elements(scores, topk)
    return out

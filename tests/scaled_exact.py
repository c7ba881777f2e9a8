"""Host emulation of the matrix the scaled models factorise, and of the dense downvote, in the reference's own arithmetic.
Shared by the CPU checks against the reference (test_oracle_scaling.py) and the device tests (test_gpu_scaled_matrix.py).

reference_csr       ``coo_matrix((val, (row, col)), shape).tocsr()`` (models.py:169-174): duplicates summed, explicit zeros
                    and duplicates that cancel kept as stored zeros.  With ``drop_zeros`` the zero triplets are filtered
                    first, as get_test_matrix does (models.py:196-201), so ``+x, -x`` still leaves a stored zero.
reference_scaled    ScaledMatrixMixin.get_training_matrix (models.py:891-895): a row pass, then a column pass, each a scipy
                    sparse product with ``diags(sqrt(count) ** (scaling - 1))`` (preprocessing/matrices.py:71-93).  The row
                    counts include the stored zeros; a sparse product stores only nonzero results, so the column counts,
                    taken after the row pass, do not -- even at row_scaling == 1, where rescale_matrix does not return
                    early.
reference_downvote  downvote_seen_items, dense branch (models.py:510-519): ``min(S) - (max(S_seen) - S_seen) - 1`` in the
                    dtype of the scores, one rounding per operation.

Summation order.  scipy sorts the indices of each row with std::sort, which is not stable, so the order in which three or
more duplicates are summed is unspecified.  reference_csr therefore only accepts duplicate runs whose sum cannot depend
on the order: pairs (a + b == b + a), and longer runs of values on a common power-of-two grid whose absolute sum fits the
significand of the input dtype (then every partial sum, in any order, is exact).  Float32 pairs must also sum exactly in
float64, so that rounding the float64 sum to float32 is what scipy's float32 addition gives."""
import fractions

import numpy as np
import scipy.sparse as sps

ULP_WIDEN = 4          # CUDA's double pow is documented to within 2 ulp; numpy's is nearly correctly rounded


def _grid_exact(vals, bits):
    """every partial sum of ``vals`` (python floats), in any order, is exact at ``bits`` significand bits."""
    q = [fractions.Fraction(v) for v in vals]
    den = max(x.denominator for x in q)             # a power of two: every value is an integer multiple of 1 / den
    return sum(abs(x) * den for x in q) < 2 ** bits


def reference_csr(idx, val, shape, drop_zeros=False):
    """float64 CSR (sorted indices) of ``coo_matrix((val, (idx[:, 0], idx[:, 1])), shape).tocsr()`` with the values the
    reference holds: for float32 feedback the float32 sums, widened to float64."""
    idx = np.asarray(idx, dtype=np.int64)
    val = np.asarray(val)
    assert val.dtype in (np.float32, np.float64), val.dtype
    bits = 24 if val.dtype == np.float32 else 53
    rows, cols = idx[:, 0], idx[:, 1]
    if drop_zeros:
        keep = val != 0
        rows, cols, val = rows[keep], cols[keep], val[keep]
    n_rows, n_cols = int(shape[0]), int(shape[1])
    key = rows * n_cols + cols
    order = np.argsort(key, kind="stable")
    key, v = key[order], val[order].astype(np.float64)
    head = np.r_[True, key[1:] != key[:-1]] if len(key) else np.zeros(0, dtype=bool)
    starts = np.flatnonzero(head)
    lengths = np.diff(np.r_[starts, len(key)])
    data = np.add.reduceat(v, starts) if len(starts) else np.zeros(0)
    for s, n in zip(starts[lengths > 1], lengths[lengths > 1]):
        run = [float(x) for x in v[s:s + n]]
        if n > 2:
            assert _grid_exact(run, bits), "duplicate run %r: its sum depends on the summation order" % (run,)
        if val.dtype == np.float32:
            assert fractions.Fraction(data[np.searchsorted(starts, s)]) == sum(map(fractions.Fraction, run)), run
    data = data.astype(val.dtype).astype(np.float64)
    ukey = key[starts]
    indptr = np.searchsorted(ukey, np.arange(n_rows + 1, dtype=np.int64) * n_cols)
    return sps.csr_matrix((data, (ukey % n_cols).astype(np.int32), indptr), shape=(n_rows, n_cols))


def scaling_factors(counts, scaling):
    """``power(sqrt(count), scaling - 1)`` for the lines with entries; 1 for empty lines (their factor multiplies nothing)."""
    norm = np.sqrt(np.asarray(counts, dtype=np.float64))
    out = np.ones_like(norm)
    nz = norm != 0
    out[nz] = np.power(norm[nz], scaling - 1)
    return out


def reference_scaled(csr, row_scaling, col_scaling):
    """ScaledMatrixMixin.get_training_matrix on the unscaled CSR ``csr`` (reference_csr).  Returns ``(values, kept, rf,
    cf)``: float64 values in the pattern of ``csr`` (entries the row pass drops are 0), whether each entry survives, and
    the row and column factors."""
    n_rows, n_cols = csr.shape
    rows = np.repeat(np.arange(n_rows), np.diff(csr.indptr))
    rf = scaling_factors(np.diff(csr.indptr), row_scaling)           # structural: stored zeros count
    v1 = csr.data * rf[rows]
    kept = v1 != 0                                                   # the row product stores only nonzero results
    cf = scaling_factors(np.bincount(csr.indices[kept], minlength=n_cols), col_scaling)
    out = np.where(kept, v1 * cf[csr.indices], 0.0)
    return out, kept, rf, cf


def _widen(f, scaling):
    """the factor's two ends ULP_WIDEN ulp apart; exact where the device computes no pow (scaling 1: factor 1)."""
    if scaling == 1:
        return f, f
    d = ULP_WIDEN * np.spacing(f)
    return f - d, f + d


def ambiguous(csr, row_scaling, col_scaling):
    """entries whose float32 result could differ with factors ULP_WIDEN ulp off numpy's: the device's ``(double)v * rf *
    cf`` (two float64 roundings, then float32) with rf and cf anywhere in the widened range lies between the two ends,
    every rounding being monotonic.  Returns ``(flag, lo, hi)``, the ends rounded to float32."""
    _, kept, rf, cf = reference_scaled(csr, row_scaling, col_scaling)
    rows = np.repeat(np.arange(csr.shape[0]), np.diff(csr.indptr))
    v = csr.data.astype(np.float32).astype(np.float64)
    r_lo, r_hi = _widen(rf[rows], row_scaling)
    c_lo, c_hi = _widen(cf[csr.indices], col_scaling)
    lo = ((v * r_lo) * c_lo).astype(np.float32)
    hi = ((v * r_hi) * c_hi).astype(np.float32)
    return kept & (lo != hi), lo, hi


def reference_downvote(S, rows, cols):
    """a lowered copy of the dense block ``S`` (the dense branch of downvote_seen_items), in S's dtype.  Repeated
    ``(row, col)`` pairs get the same value: every new value is computed from the scores before the write."""
    S = np.array(S, copy=True)
    one = S.dtype.type(1)
    seen = S[rows, cols]
    mn, mx = S.min(), seen.max()
    S[rows, cols] = (mn - (mx - seen)) - one
    return S


def feedback_case(seed, n_rows=60, n_cols=40, dtype=np.float32, sorted_input=False, representable=True):
    """Triplets ``(idx [nnz x 2] int64, val)`` of feedback with what the scaling gets wrong if it counts stored zeros:
    non-integer values, explicit 0.0 and -0.0, duplicate pairs that cancel, row 1 made only of zeros, column 2 whose only
    entries are zeros, empty rows and columns (the last two of each), and row 0 longer than 32 entries.  Unsorted input
    also has duplicate pairs that add up and duplicate triples of dyadic values, and comes shuffled (the ingest's sort
    path); ``sorted_input`` gives strictly increasing unique (row, col) (its fast path).  ``representable=False`` gives
    float64 values float32 cannot hold (float64 only)."""
    rng = np.random.default_rng(seed)
    used_rows, used_cols = n_rows - 2, n_cols - 2
    dense = rng.random((used_rows, used_cols)) < 0.25
    dense[0, :] = True                                         # the long row: more than 32 entries
    dense[0, rng.choice(used_cols, 3, replace=False)] = False
    dense[1, :] = False
    dense[1, [0, 3, 5]] = True                                 # row 1: zeros only (set below)
    dense[:, 2] = False
    dense[[0, 4, 7], 2] = True                                 # column 2: zeros only (set below)
    r, c = np.nonzero(dense)
    if representable:
        v = rng.uniform(0.3, 5.0, len(r)).astype(np.float32).astype(np.float64)
    else:
        v = rng.integers(3, 50, len(r)) / 10.0                 # 0.3, 0.4, ...: most are not float32 values
    z = rng.random(len(r)) < 0.12
    v[z] = 0.0
    v[z & (rng.random(len(r)) < 0.5)] = -0.0
    v[(r == 1) | (c == 2)] = 0.0
    v[(r == 1) & (c == 5)] = -0.0
    v[0] = -0.0
    rows, cols, vals = [r], [c], [v]
    if not sorted_input:
        pick = rng.choice(len(r), len(r) // 6, replace=False)
        half = len(pick) // 2
        cancel, add = pick[:half], pick[half:]
        rows += [r[cancel], r[add]]
        cols += [c[cancel], c[add]]
        w = rng.uniform(0.3, 5.0, len(add)).astype(np.float32).astype(np.float64) if representable \
            else rng.integers(3, 50, len(add)) / 10.0
        vals += [-v[cancel], w]
        # a cancelling pair in the zero row and one in the zero column, then dyadic triples
        rows += [np.array([1, 1, 4]), np.array([1, 1, 4])]
        cols += [np.array([7, 7, 2]), np.array([7, 7, 2])]
        vals += [np.array([1.75, -1.75, 0.5]), np.array([0.0, 0.0, -0.5])]
        tri = rng.choice(np.setdiff1d(np.arange(len(r)), pick), 5, replace=False)
        for t in tri:
            rows.append(np.full(2, r[t]))
            cols.append(np.full(2, c[t]))
            vals.append(np.array([0.25, -0.625]))
            v[t] = 1.5                                         # dyadic head of the triple
    rows, cols, vals = np.concatenate(rows), np.concatenate(cols), np.concatenate(vals)
    if sorted_input:
        order = np.lexsort((cols, rows))
    else:
        order = rng.permutation(len(rows))
    idx = np.stack([rows[order], cols[order]], axis=1).astype(np.int64)
    return idx, vals[order].astype(dtype)

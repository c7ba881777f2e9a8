"""Host emulation of the scoring contract (DESIGN.md §3.1, §4 "Scoring"), shared by the exact scoring tests.

canonical_scores   the canonical fp32 score of every (user, item) pair: s = fmaf(e[r-1], v[r-1], ... fmaf(e[0], v[0], 0))
                   with one rounding per step, IEEE subnormals and signed zeros (the library is built without fast-math);
expected_lists     the reference lists: unseen items by (score desc, id asc), -0 equal to +0, then -- when fewer than k are
                   unseen -- the seen items in the same order; NaN never enters, empty slots are {-1, -inf};
expected_cands     one item shard's candidate lists: unseen items only, global ids.

fmaf32 forms fmaf(a, b, c) exactly for arbitrary fp32 data: a*b is exact in float64, c is added with TwoSum, the float64
sum is rounded to odd and then cast to float32 (correct because 53 >= 24 + 2, also where the result is subnormal).  An
exact zero keeps the sign IEEE gives a*b + c (-0 only when both are -0), which the float64 add already does."""
import fractions

import numpy as np

FULL_EMULATION_STEPS = 20_000_000      # pair-steps (m * n * r) emulated step by step; larger cases must be dyadic


def fmaf32(a, b, c):
    """fmaf on float32 arrays (broadcasting): a*b + c rounded once to float32, round to nearest even."""
    p = np.asarray(a, np.float64) * np.asarray(b, np.float64)        # exact: 24 + 24 significant bits
    cd = np.asarray(c, np.float64)
    s = p + cd
    bp = s - p
    err = (p - (s - bp)) + (cd - bp)                                  # TwoSum: p + c == s + err exactly
    bits = np.ascontiguousarray(s).view(np.int64)
    # round to odd: an inexact sum with an even last bit moves to its odd neighbour on the side of the exact value
    fix = (err != 0) & ((bits & 1) == 0)
    away = (err > 0) == (s > 0)                                       # |p + c| > |s|
    bits = bits + np.where(fix, np.where(away, 1, -1), 0)
    return bits.view(np.float64).astype(np.float32)


def round_fraction_f32(q, zero_sign=1):
    """Fraction -> nearest float32, ties to even (finite range, subnormals included).  An exact zero gets ``zero_sign``;
    a nonzero value that rounds to zero keeps its own sign."""
    if q == 0:
        return np.float32(0.0) if zero_sign > 0 else np.float32(-0.0)
    sign = -1 if q < 0 else 1
    q = abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if fractions.Fraction(2) ** e > q:
        e -= 1
    ulp = fractions.Fraction(2) ** (max(e, -126) - 23)
    n, rem = divmod(q, ulp)
    half = fractions.Fraction(1, 2) * ulp
    if rem > half or (rem == half and n % 2 == 1):
        n += 1
    return np.float32(sign * float(n * ulp))


def fmaf_fraction(a, b, c):
    """reference fmaf of three float32 scalars in rational arithmetic, one rounding, IEEE zero signs"""
    F = fractions.Fraction
    a, b, c = np.float32(a), np.float32(b), np.float32(c)
    exact = F(float(a)) * F(float(b)) + F(float(c))
    prod_neg_zero = (a == 0 or b == 0) and (np.signbit(a) != np.signbit(b))
    both_neg_zero = c == 0 and np.signbit(c) and prod_neg_zero
    return round_fraction_f32(exact, -1 if both_neg_zero else 1)


def _dyadic_unit(x):
    """per row: the largest power of two every entry is an integer multiple of (inf for an all-zero row)"""
    x = np.asarray(x, np.float32)
    mant, ex = np.frexp(x.astype(np.float64))
    mi = np.abs(mant * 2.0 ** 24).astype(np.int64)                    # 24-bit integer significand
    lowest_bit = np.where(mi != 0, mi & -mi, 1).astype(np.float64)
    low = np.where(mi != 0, np.log2(lowest_bit), np.inf)
    return np.min(ex - 24 + low, axis=1)


def canonical_scores(E, V, r):
    """[m x n] float32: the canonical score of every (row of E, row of V) pair over the first r columns (later columns are
    never read, so they may hold anything, NaN included).  Up to FULL_EMULATION_STEPS pair-steps every fmaf is emulated;
    beyond that the factors must be dyadic (every partial sum exact in fp32), which is asserted, and then the float64
    product rounded once is the canonical score."""
    E = np.ascontiguousarray(np.asarray(E, np.float32)[:, :r])
    V = np.ascontiguousarray(np.asarray(V, np.float32)[:, :r])
    m, n = E.shape[0], V.shape[0]
    if m * n * r <= FULL_EMULATION_STEPS:
        s = np.zeros((m, n), np.float32)
        for t in range(r):
            s = fmaf32(E[:, t, None], V[None, :, t], s)
        return s
    ue, uv = _dyadic_unit(E), _dyadic_unit(V)
    unit = ue[:, None] + uv[None, :]                                  # log2 of the unit of every partial sum
    bound = np.abs(E).astype(np.float64) @ np.abs(V).astype(np.float64).T
    live = bound > 0
    assert np.all(unit[live] >= -149), "dyadic factors below the subnormal grid: scores would round"
    assert np.all(bound[live] < np.exp2(unit[live] + 24)), "dyadic factors too wide: partial sums would round"
    # every fmaf is exact, so the chain is the exact sum; a zero is +0 (the chain starts at +0 and nothing underflows)
    return ((E.astype(np.float64) @ V.astype(np.float64).T) + 0.0).astype(np.float32)


def _seen_sets(seen, m):
    if seen is None:
        return [np.zeros(0, np.int64)] * m
    indptr, indices = np.asarray(seen[0]), np.asarray(seen[1])
    return [np.asarray(indices[indptr[u]:indptr[u + 1]], np.int64) for u in range(m)]


def _order(scores, ids):
    """positions of ``ids`` by (score desc, id asc), -0 == +0, NaN left out"""
    ok = ~np.isnan(scores)
    s, i = scores[ok] + scores.dtype.type(0.0), ids[ok]             # -0 + 0 = +0: the two zeros tie
    return np.flatnonzero(ok)[np.lexsort((i, -s.astype(np.float64)))]


def expected_lists(S32, seen, k, item_offset=0, fill=True):
    """(ids int64 [m x k], scores float32 [m x k]) of the reference order for the score block S32 [m x n] whose column j is
    the item with global id j + item_offset; ``seen`` = (indptr, indices) of global ids or None.  With ``fill`` the seen
    items follow when fewer than k are unseen.  A float64 block keeps its type (pb200_topk_dense)."""
    S32 = np.asarray(S32)
    if S32.dtype != np.float64:
        S32 = S32.astype(np.float32)
    m, n = S32.shape
    ids_out = np.full((m, k), -1, np.int64)
    sc_out = np.full((m, k), -np.inf, S32.dtype)
    gid = np.arange(n, dtype=np.int64) + item_offset
    for u, seen_u in enumerate(_seen_sets(seen, m)):
        is_seen = np.isin(gid, seen_u)
        unseen = np.flatnonzero(~is_seen)
        pick = unseen[_order(S32[u, unseen], gid[unseen])]
        if fill and len(pick) < k:
            was = np.flatnonzero(is_seen)
            pick = np.concatenate([pick, was[_order(S32[u, was], gid[was])]])
        pick = pick[:k]
        ids_out[u, :len(pick)] = gid[pick]
        sc_out[u, :len(pick)] = S32[u, pick]
    return ids_out, sc_out


def expected_cands(S32, seen, k, item_offset=0):
    """one shard's candidate lists (pb200_score_topk_cands): unseen items only, global ids, {-1, -inf} padding"""
    return expected_lists(S32, seen, k, item_offset, fill=False)


def csr_of(rows_of_ids, m):
    """(indptr int64, indices int32) of per-row id collections (sorted, unique)"""
    rows = [np.unique(np.asarray(rows_of_ids[u], np.int64)) if u < len(rows_of_ids) else np.zeros(0, np.int64)
            for u in range(m)]
    indptr = np.zeros(m + 1, np.int64)
    indptr[1:] = np.cumsum([len(x) for x in rows])
    indices = np.concatenate(rows).astype(np.int32) if indptr[-1] else np.zeros(0, np.int32)
    return indptr, indices

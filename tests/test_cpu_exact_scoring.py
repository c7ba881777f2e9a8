"""The host emulation of the scoring contract (tests/exact_scoring.py) against rational arithmetic and hand-built lists.
CPU only: the GPU scoring tests compare the kernels with this emulation bit for bit, so it has to be right first."""
import fractions

import numpy as np
import pytest

from tests.exact_scoring import (canonical_scores, csr_of, expected_cands, expected_lists, fmaf32, fmaf_fraction,
                                 round_fraction_f32)

F = fractions.Fraction


def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def _chain_fraction(e, v):
    s = np.float32(0.0)
    for a, b in zip(e, v):
        s = fmaf_fraction(a, b, s)
    return s


def _rand_f32(rng, n, lo, hi):
    mant = rng.integers(0, 1 << 23, n).astype(np.uint32)
    exp = rng.integers(lo + 127, hi + 127, n).astype(np.uint32)
    sign = rng.integers(0, 2, n).astype(np.uint32) << np.uint32(31)
    return (sign | (exp << np.uint32(23)) | mant).view(np.float32)


def test_fmaf_matches_rational_arithmetic_at_the_edges():
    """single fmaf steps: subnormal operands and results, products that underflow to +-0, exact cancellation to +0,
    every combination of signed zeros, and magnitudes near 2^120"""
    rng = np.random.default_rng(3)
    tiny = np.float32(2.0 ** -149)
    sub = (rng.integers(1, 1 << 23, 200).astype(np.uint32) |
           (rng.integers(0, 2, 200).astype(np.uint32) << np.uint32(31))).view(np.float32)
    assert sub.shape == (200,) and np.all(np.abs(sub) < np.float32(2.0 ** -126))
    a = [sub, _rand_f32(rng, 200, -80, -70), _rand_f32(rng, 200, 55, 62), _rand_f32(rng, 200, -5, 5)]
    b = [_rand_f32(rng, 200, -3, 3), _rand_f32(rng, 200, -80, -70), _rand_f32(rng, 200, 55, 62), _rand_f32(rng, 200, -5, 5)]
    c = [rng.permutation(sub),np.where(rng.random(200) < 0.5, np.float32(0.0), np.float32(-0.0)),
         _rand_f32(rng, 200, 118, 122), np.zeros(200, np.float32)]
    # exact cancellation: c = -a*b where the product is representable
    x, y = rng.integers(-100, 100, 100).astype(np.float32), rng.integers(-100, 100, 100).astype(np.float32)
    a.append(x); b.append(y); c.append(-(x * y))
    zeros = np.array([0.0, -0.0], np.float32)
    za, zb, zc = (g.ravel() for g in np.meshgrid(np.concatenate([zeros, [1.0, -1.0, tiny, -tiny]]).astype(np.float32),
                                                 np.concatenate([zeros, [2.0 ** -100, -(2.0 ** -100)]]).astype(np.float32),
                                                 zeros, indexing="ij"))
    a.append(za); b.append(zb); c.append(zc)
    A, B, C = (np.concatenate(t).astype(np.float32) for t in (a, b, c))
    got = fmaf32(A, B, C)
    ref = np.array([fmaf_fraction(p, q, s) for p, q, s in zip(A, B, C)], np.float32)
    np.testing.assert_array_equal(_bits(got), _bits(ref))
    # the cases do reach the edges they are meant to
    assert (got == 0).any() and (np.signbit(got) & (got == 0)).any() and (~np.signbit(got) & (got == 0)).any()
    assert ((np.abs(got) < np.float32(2.0 ** -126)) & (got != 0)).any()
    assert (np.abs(got) > np.float32(2.0 ** 119)).any()


def test_canonical_scores_match_rational_chains():
    """whole chains (every step rounded once) against Fraction arithmetic: ordinary data, rows scaled to 2^-70 so that
    products underflow and the score is a signed zero or subnormal, rows near 2^60 (scores near 2^120), subnormal factor
    entries; columns beyond r hold NaN and must not be read"""
    rng = np.random.default_rng(5)
    r = 7
    E = rng.standard_normal((6, r + 2)).astype(np.float32)
    V = rng.standard_normal((9, r + 2)).astype(np.float32)
    E[1] = (rng.integers(-2, 3, r + 2) * 2.0 ** -76).astype(np.float32)       # products ~2^-152: round to +-0
    V[2] = (rng.integers(-2, 3, r + 2) * 2.0 ** -76).astype(np.float32)
    E[2] *= np.float32(2.0 ** 60)
    V[3] *= np.float32(2.0 ** 59)
    E[3] = (rng.integers(1, 1 << 20, r + 2) * 2.0 ** -149 * rng.choice([-1, 1], r + 2)).astype(np.float32)   # subnormal
    E[4] *= np.float32(2.0 ** -70)
    V[4] *= np.float32(2.0 ** -60)
    E[5] = 0.0
    E[:, r:] = np.nan
    V[:, r:] = np.nan
    got = canonical_scores(E, V, r)
    ref = np.array([[_chain_fraction(E[u, :r], V[j, :r]) for j in range(V.shape[0])] for u in range(E.shape[0])], np.float32)
    np.testing.assert_array_equal(_bits(got), _bits(ref))
    assert not np.isnan(got).any()
    assert (np.signbit(got) & (got == 0)).any()                # a -0 score is among them
    assert (np.abs(got) > np.float32(2.0 ** 110)).any()


def test_dyadic_shortcut_equals_the_chain(monkeypatch):
    """above the full-emulation size the dyadic shortcut is used: on dyadic data it must equal the step-by-step chain, and
    data that would round must be refused"""
    import tests.exact_scoring as xs
    rng = np.random.default_rng(9)
    E = (rng.integers(-2, 3, (40, 20)) * 2.0 ** -3).astype(np.float32)
    V = (rng.integers(-2, 3, (70, 20)) * 2.0 ** 5).astype(np.float32)
    E[3] *= np.float32(2.0 ** -30)                               # per-row scales are fine
    full = canonical_scores(E, V, 20)
    monkeypatch.setattr(xs, "FULL_EMULATION_STEPS", 0)
    np.testing.assert_array_equal(_bits(canonical_scores(E, V, 20)), _bits(full))
    with pytest.raises(AssertionError):
        canonical_scores(rng.standard_normal((4, 20)).astype(np.float32), V, 20)


def test_round_fraction_keeps_the_sign_of_an_underflow():
    assert np.signbit(round_fraction_f32(F(-1, 2 ** 160)))
    assert not np.signbit(round_fraction_f32(F(0)))
    assert np.signbit(round_fraction_f32(F(0), -1))
    assert round_fraction_f32(F(3, 2 ** 150)) == np.float32(2.0 ** -148)        # 1.5 ulp of the subnormal grid: to even


def test_expected_lists_on_hand_built_rows():
    S = np.array([
        [1.0, 2.0, 2.0, 0.0, -0.0, 3.0],                   # ties: id asc; -0 and +0 tie
        [-0.0, 0.0, -0.0, 0.0, -1.0, -np.inf],             # all zeros of both signs
        [np.nan, 5.0, np.nan, -np.inf, 1.0, 1.0],          # NaN never enters; -inf is a score like any other
        [4.0, 3.0, 2.0, 1.0, 0.0, -1.0],                   # fewer than k unseen: seen ones follow, best first
        [1.0, 1.0, 1.0, 1.0, 1.0, 1.0],                    # everything seen
    ], np.float32)
    seen = csr_of([[0], [], [1], [0, 2, 3, 5], [0, 1, 2, 3, 4, 5]], 5)
    ids, sc = expected_lists(S, seen, 4)
    np.testing.assert_array_equal(ids, [[5, 1, 2, 3], [0, 1, 2, 3], [4, 5, 3, 1], [1, 4, 0, 2], [0, 1, 2, 3]])
    assert _bits(sc[1]).tolist() == _bits(np.array([-0.0, 0.0, -0.0, 0.0], np.float32)).tolist()   # signs kept
    assert sc[2, 2] == -np.inf and ids[2, 2] == 3
    ids, sc = expected_lists(S, seen, 6, item_offset=0)
    np.testing.assert_array_equal(ids[2], [4, 5, 3, 1, -1, -1])   # two NaN: padding
    assert np.all(sc[2, 4:] == -np.inf)
    # candidate lists of a shard: unseen only, global ids
    ids, sc = expected_cands(S[:, 2:], seen, 4, item_offset=2)
    np.testing.assert_array_equal(ids, [[5, 2, 3, 4], [2, 3, 4, 5], [4, 5, 3, -1], [4, -1, -1, -1], [-1, -1, -1, -1]])
    assert np.all(sc[4] == -np.inf)

"""The host emulation of the CoFFee build kernels (tests/hooi_exact.py) against literal walks of the kernels' loops and
against the f64 bounds of tests/test_gpu_hooi.py, and its fixtures against the orders the kernels do not use: each
alternative order must change the bits of a stated number of output entries.  No GPU needed."""
import numpy as np
import pytest

from oracle import polara_oracle as po
from tests import hooi_exact as he
from tests.test_gpu_hooi import _ttm_gamma, _xgram_ref

# rows that end on, one before and one after a window, carried over several windows, past the long-row cutoff and empty
SMALL_ROWS = [0, 3, 513, 1, 2, 0, 0, 1100, 4697, 29, 5, 511, 0, 31, 33, 1, 0, 9, 0]
SMALL_SEGMENTS = [0, 3100, 40, 33, 0, 1024, 65]


def _bits_equal(x, y):
    np.testing.assert_array_equal(np.asarray(x, np.float32).view(np.int32), np.asarray(y, np.float32).view(np.int32))


def _grouped(lengths, ru, rw, seed, **kw):
    idx, val, u, w = he.ttm_fixture(lengths, ru, rw, seed, **kw)
    return idx, val, u, w, he.group(idx, val, len(lengths))


@pytest.mark.parametrize("kind", ["window", "ldg"])
def test_ttm_emulation_matches_the_kernel_walk(kind):
    """bit for bit against the scalar walk; within the f64 bound of test_gpu_hooi.py; empty rows +0"""
    ru, rw = 3, 5
    idx, val, u, w, (seg, i1, i2, v) = _grouped(SMALL_ROWS, ru, rw, 0, n1=300, n2=200)
    got = he.ttm(kind, seg, i1, i2, v, u, w, ru, rw)
    _bits_equal(got, he.walk_ttm(kind, seg, i1, i2, v, u, w, ru, rw))
    empty = np.asarray(SMALL_ROWS) == 0
    assert not got[empty].any() and not np.signbit(got[empty]).any()
    shape = (len(SMALL_ROWS), 300, 200)
    u64, w64 = u[:, :ru].astype(np.float64), w[:, :rw].astype(np.float64)
    ref = po.ttm3d(idx, val.astype(np.float64), shape, u64, w64, 0, 1, 2).reshape(shape[0], -1)
    scale = po.ttm3d(idx, np.abs(val).astype(np.float64), shape, np.abs(u64), np.abs(w64), 0, 1, 2)
    scale = scale.reshape(shape[0], -1)
    gamma = _ttm_gamma(SMALL_ROWS, kind, ru * rw)[:, None]
    assert (np.abs(got - ref) <= gamma * scale).all()


def test_ttm_emulation_of_a_row_subset():
    """``rows=`` gives exactly those rows of the full output"""
    ru, rw = 2, 3
    _, _, u, w, (seg, i1, i2, v) = _grouped(SMALL_ROWS, ru, rw, 1, n1=300, n2=200)
    rows = np.array([8, 2, 0, 7])
    for kind in ("window", "ldg"):
        full = he.ttm(kind, seg, i1, i2, v, u, w, ru, rw)
        _bits_equal(he.ttm(kind, seg, i1, i2, v, u, w, ru, rw, rows=rows), full[rows])


@pytest.mark.parametrize("num_sms", [1, 132])
def test_ttm_reduce_emulation_matches_the_kernel_walk(num_sms):
    """bit for bit against the scalar walk over 64 x 64 tiles (here 2 x 1), with one block per segment (num_sms = 1 caps
    it at 2) or ceil(len / 1024); within the f64 bound of test_gpu_hooi.py"""
    ra, rb = 66, 2
    seg, ia, ib, val, a, b = he.reduce_fixture(SMALL_SEGMENTS, ra, rb, 1, na=100, nb=90)
    got = he.ttm_reduce(seg, ia, ib, val, a, b, ra, rb, num_sms)
    _bits_equal(got, he.walk_ttm_reduce(seg, ia, ib, val, a, b, ra, rb, num_sms))
    assert not got[np.asarray(SMALL_SEGMENTS) == 0].any()
    ref, scale = _xgram_ref(seg, ia, ib, val, a, b)
    assert (np.abs(got - ref) <= 2.0 ** -22 * (scale + np.abs(ref))).all()


def test_reduce_blocks():
    """pb200_ttm_reduce's blocking: ceil(len / 1024) blocks capped at 2 * num_sms, rows per block a multiple of 32"""
    assert he.reduce_blocks(0, 132) == (1, 32)
    assert he.reduce_blocks(1, 132) == (1, 32)
    assert he.reduce_blocks(1024, 132) == (1, 1024)
    assert he.reduce_blocks(1025, 132) == (2, 544)
    assert he.reduce_blocks(3 * 1024, 132) == (3, 1024)
    assert he.reduce_blocks(300_001, 132) == (261, 1152)
    assert he.reduce_blocks(300_001, 114) == (224, 1344)
    assert he.reduce_blocks(2 * 132 * 1024 + 77, 132) == (257, 1056)     # past the cap: fewer blocks once rounded


def _count(x, y):
    return int(he.differs(x, y).sum())


# rows around the window and long-row boundaries, the short rows of the width sweep and one long row of 9000 nnz
ORDER_ROWS = he.TTM_EDGES["window_bounds"] + he.TTM_EDGES["long_row_cutoff"] + list(he.WIDTH_ROWS[:120]) + [9000]
# per alternative: the least number of entries (of 140 x 15) whose bits must differ from the contract
TTM_LEAST = {"window": {"desc": 400, "win1024": 30, "carries_rev": 20, "fma_vuw": 350, "unfused": 200},
             "ldg": {"desc": 400, "fma_vuw": 350, "unfused": 200, "warps_rev": 10, "no_split": 15}}


@pytest.mark.parametrize("kind", ["window", "ldg"])
def test_the_ttm_fixture_tells_the_orders_apart(kind, capsys):
    ru, rw = 3, 5
    _, _, u, w, (seg, i1, i2, v) = _grouped(ORDER_ROWS, ru, rw, 11)
    base = he.ttm(kind, seg, i1, i2, v, u, w, ru, rw)
    counts = {alt: _count(base, he.ttm(kind, seg, i1, i2, v, u, w, ru, rw, alt=alt)) for alt in TTM_LEAST[kind]}
    with capsys.disabled():
        print("\n%s: entries that differ from the contract of %d: %s" % (kind, base.size, counts))
    for alt, least in TTM_LEAST[kind].items():
        assert counts[alt] >= least, (alt, counts[alt])


# one segment past the block cap at 114 and at 132 SMs, segments of k * 1024 and 32 j +- 1 nnz, empty ones
ORDER_SEGMENTS = [0, 300_001, 3 * 1024, 5 * 1024, 1023, 1025, 31, 33, 63, 65, 0, 4097, 0, 2000]
# per alternative: the least number of entries (of 14 x 30) whose bits must differ from the contract at 132 SMs
REDUCE_LEAST = {"va64": 90, "blocks_rev": 15, "partial32": 200, "sms114": 12}


def test_the_reduce_fixture_tells_the_orders_apart(capsys):
    ra, rb = 5, 6
    seg, ia, ib, val, a, b = he.reduce_fixture(ORDER_SEGMENTS, ra, rb, 2)
    base = he.ttm_reduce(seg, ia, ib, val, a, b, ra, rb, 132)
    counts = {alt: _count(base, he.ttm_reduce(seg, ia, ib, val, a, b, ra, rb, 132, alt=alt)) for alt in REDUCE_LEAST}
    with capsys.disabled():
        print("\nttm_reduce: entries that differ from the contract of %d: %s" % (base.size, counts))
    for alt, least in REDUCE_LEAST.items():
        assert counts[alt] >= least, (alt, counts[alt])


def test_the_reduce_fixture_has_its_structure():
    """a segment of more than 1024 nnz holds N_BIG large pairs that cancel exactly, and at 114 and at 132 SMs the halves
    of at least two pairs lie in different row blocks; shorter segments hold no large term"""
    seg, ia, ib, val, a, b = he.reduce_fixture(ORDER_SEGMENTS, 5, 6, 2)
    for s, n in enumerate(ORDER_SEGMENTS):
        lo, hi = seg[s], seg[s + 1]
        big = lo + np.flatnonzero(ia[lo:hi] < he.N_BIG)
        assert len(big) == (2 * he.N_BIG if n > he.REDUCE_ROWS else 0)
        split = {114: 0, 132: 0}
        for k in range(he.N_BIG if n > he.REDUCE_ROWS else 0):
            p, q = big[ia[big] == k]
            assert ib[p] == ib[q] == k and val[p] == -val[q]
            for sms in split:
                rpb = he.reduce_blocks(n, sms)[1]
                split[sms] += (p - lo) // rpb != (q - lo) // rpb
        assert n <= he.REDUCE_ROWS or min(split.values()) >= 2, (n, split)
    assert np.abs(a[:he.N_BIG]).min() >= 2.0 ** 20 and np.abs(a[he.N_BIG:]).max() < 2.0 ** 5

"""The kernels of the CoFFee build (CoffeeModel.build -> _hooi_device) against float64 host references on every code path
they have and at CoFFee ranks: pb200_ttm (csrc/hooi.cu), pb200_ttm_reduce (csrc/hooi.cu), pb200_coo_group
(csrc/csr_ops.cu), pb200_tall_svd (csrc/rsvd.cu) on the buffers HOOI hands it, and one whole HOOI build.  H100 only.

Tolerances follow from each kernel's summation order (DESIGN.md §4):
  * fp32 ``fmaf`` chains (pb200_ttm): ``|got - ref| <= gamma * scale`` where ``scale`` is the same contraction of |val|,
    |U|, |W|; gamma = 5e-6 for rows of up to LONG_ROW nnz and ``2^-24 * depth`` for longer rows, depth being the longest
    chain of roundings the kernel's order implies (window kernel: 512 per window + one per carried piece; row-owned kernel:
    len / 8 per warp + the 8 warp partials).
  * fp64 accumulation (pb200_ttm_reduce, the Gram matrix of pb200_tall_svd): ``2^-22 * (scale + |ref|)``.
  * every kernel is deterministic: a second run is bit-identical.

These bounds catch a lost window piece or warp partial, not a wrong summation order.  The order itself is checked bit for
bit against the host emulation of tests/hooi_exact.py in tests/test_gpu_hooi_exact.py (the kernels, the products of a
real build and the CoFFee lists) and tests/test_cpu_hooi_exact.py (the emulation and its fixtures)."""
import functools

import numpy as np
import pytest
import torch

from oracle import polara_oracle as po
from tests.helpers import check_topk_against_scores, subspace_gap
from tests.hooi_exact import TTM_EDGES, WIDTH_ROWS

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24                               # unit roundoff of float32
GAMMA_SHORT = 5e-6                             # fmaf chains of up to a few thousand terms (as in the SpMM tests)
TW, CB, LONG_ROW, WARPS = 512, 2048, 4096, 8   # window size, row-owned block size, long-row cutoff, warps (csrc/hooi.cu)


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    return get_engine(0)


@pytest.fixture(params=["window", "ldg"])
def ttm_kernel(request, eng):
    """"window": nnz windows per warp + carried row pieces (width <= 512); "ldg": the row-owned kernel, which is also
    what every switch value runs for width > 512 ("bulk" / "cpasync" take the ldg path, "window32" the window path)."""
    eng.set_spmm_kernel(request.param)
    yield request.param
    eng.set_spmm_kernel("window")


def _ttm(eng, n0, seg, i1, i2, val, u, ru, w, rw):
    """``Engine.ttm`` into an output that starts as NaN rather than as whatever ``empty()`` returns: an entry the kernel
    never writes cannot pass for a right value left in that memory by an earlier call."""
    from polara_b200.engine import _p, round_up
    ldo = round_up(ru * rw, 4)
    out = torch.full((n0, ldo), float("nan"), dtype=torch.float32, device=eng.device)
    st = eng.lib.pb200_ttm(eng.h, n0, i1.shape[0], _p(seg, torch.int64), _p(i1, torch.int32), _p(i2, torch.int32),
                           _p(val, torch.float32), _p(u, torch.float32), ru, u.stride(0), _p(w, torch.float32), rw,
                           w.stride(0), _p(out), ldo)
    eng._check(st, "ttm")
    return out


def _factor(rng, n, r, pad):
    """[n x r] float32 factor stored as the leading columns of an [n x (r + pad)] array (odd leading dimensions).  Entries
    in [-0.5, 1): signs mix, but every contraction has a nonzero mean, so a lost window piece or warp partial shifts the
    result by about its own size instead of by a random-walk fraction of it."""
    full = rng.uniform(-0.5, 1.0, size=(n, r + pad)).astype(np.float32)
    return full, full[:, :r]


@functools.lru_cache(maxsize=None)
def _ttm_case(lengths, ru, rw, seed):
    """COO tensor whose mode-0 segments have the given lengths, in shuffled (ungrouped) order, its factors, and the f64
    reference ``po.ttm3d`` with the ``scale`` of the tolerance (the same contraction of absolute values)."""
    rng = np.random.default_rng(seed)
    lengths = np.asarray(lengths, dtype=np.int64)
    n0, n1, n2 = len(lengths), 3000, 2000
    nnz = int(lengths.sum())
    key = np.repeat(np.arange(n0), lengths)[rng.permutation(nnz)]
    idx = np.stack([key, rng.integers(0, n1, nnz), rng.integers(0, n2, nnz)], axis=1)
    val = rng.integers(1, 6, size=nnz).astype(np.float32)
    u_full, u = _factor(rng, n1, ru, 3)
    w_full, w = _factor(rng, n2, rw, 1)
    shape = (n0, n1, n2)
    u64, w64 = u.astype(np.float64), w.astype(np.float64)
    ref = po.ttm3d(idx, val.astype(np.float64), shape, u64, w64, 0, 1, 2).reshape(n0, ru * rw)
    scale = po.ttm3d(idx, np.abs(val).astype(np.float64), shape, np.abs(u64), np.abs(w64), 0, 1, 2).reshape(n0, ru * rw)
    return idx, val, u_full, w_full, ref, scale


def _ttm_gamma(lengths, kernel, width):
    """per-row bound factor of pb200_ttm (see the module docstring)."""
    lengths = np.asarray(lengths, dtype=np.int64)
    if kernel == "window" and width <= 512:
        depth = TW + lengths // TW + 2                 # one chain per window, then the carried pieces in window order
    else:
        depth = -(-lengths // WARPS) + WARPS           # long rows: one chain per warp, then the 8 warp partials
    return np.where(lengths <= LONG_ROW, GAMMA_SHORT, np.maximum(GAMMA_SHORT, depth * U32))


def _run_ttm_case(eng, kernel, lengths, ru, rw, seed=0):
    """Groups the tensor with eng.coo_group exactly as _hooi_device does, runs pb200_ttm twice and checks the result against
    the f64 reference; returns the output for further comparisons."""
    lengths = tuple(int(x) for x in lengths)
    idx, val, u_full, w_full, ref, scale = _ttm_case(lengths, ru, rw, seed)
    n0, width = len(lengths), ru * rw
    key, a, b = (eng.upload(idx[:, c].astype(np.int32)) for c in range(3))
    seg, ao, bo, vo = eng.coo_group(key, n0, a, b, eng.upload(val))
    u_d, w_d = eng.upload(u_full)[:, :ru], eng.upload(w_full)[:, :rw]
    out = _ttm(eng, n0, seg, ao, bo, vo, u_d, ru, w_d, rw)[:, :width]
    got = out.cpu().numpy().astype(np.float64)
    empty = np.asarray(lengths) == 0
    assert not got[empty].any(), "rows of empty segments must be written as exact zeros"
    assert np.isfinite(got).all(), "an output entry was never written"
    gamma = _ttm_gamma(lengths, kernel, width)[:, None]
    ratio = np.abs(got - ref) / np.maximum(gamma * scale, 1e-300)
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert ratio[worst] <= 1.0, "row %d (%d nnz), column %d: |err| = %.3g x bound" % (
        worst[0], lengths[worst[0]], worst[1], ratio[worst])
    again = _ttm(eng, n0, seg, ao, bo, vo, u_d, ru, w_d, rw)[:, :width]
    assert torch.equal(out, again), "pb200_ttm is not deterministic"
    return out


@pytest.mark.parametrize("ru,rw", [(3, 2), (5, 24), (4, 32), (3, 43), (4, 60), (4, 64), (3, 86), (4, 128), (5, 103),
                                   (32, 32)])
def test_ttm_widths_match_f64(eng, ttm_kernel, ru, rw):
    """Every template instance of both TTM kernels: ttm_window_kernel<4|8|16> (width <= 128, <= 256, <= 512) and
    ttm_kernel<4|8|16|32>; the widths sit on and just past each boundary (128 / 129, 256 / 258, 512 / 515) and include the
    C4 mode-0 width 240.  Factors are column slices (ldu = ru + 3, ldw = rw + 1)."""
    out = _run_ttm_case(eng, ttm_kernel, WIDTH_ROWS, ru, rw)
    if ru * rw > 512:
        # beyond 512 columns every switch value runs the row-owned kernel: the other value must give the same bits
        eng.set_spmm_kernel("ldg" if ttm_kernel == "window" else "window")
        other = _run_ttm_case(eng, ttm_kernel, WIDTH_ROWS, ru, rw)
        assert torch.equal(out, other)


def test_ttm_rejects_more_than_1024_columns(eng):
    z32 = eng.upload(np.zeros(4, dtype=np.int32))
    seg = eng.upload(np.array([0, 4], dtype=np.int64))
    u = eng.upload(np.ones((1, 33), dtype=np.float32))
    w = eng.upload(np.ones((1, 32), dtype=np.float32))
    with pytest.raises(ValueError):
        eng.ttm(1, seg, z32, z32, eng.upload(np.ones(4, dtype=np.float32)), u, 33, w, 32)


@pytest.mark.parametrize("case", sorted(TTM_EDGES))
@pytest.mark.parametrize("ru,rw", [(4, 60), (3, 2)])
def test_ttm_segment_edges_match_f64(eng, ttm_kernel, case, ru, rw):
    """Rows that end on, one before or one after a window / block boundary, rows carried across many windows (the fixup
    kernel), rows split over the 8 warps, empty rows everywhere (including the tail loop after the last nnz), and an
    empty tensor: values against f64, empty rows as exact zeros, deterministic."""
    _run_ttm_case(eng, ttm_kernel, TTM_EDGES[case], ru, rw, seed=3)


# ---------------------------------------------------------------------------------------------------------------------
#  pb200_ttm_reduce
# ---------------------------------------------------------------------------------------------------------------------
def _xgram_ref(seg, ia, ib, val, a, b):
    """out[s] = A[ia]^T diag(val) B[ib] over segment s in float64, and the same of the absolute values."""
    n_seg = len(seg) - 1
    ref = np.zeros((n_seg, a.shape[1] * b.shape[1]))
    scale = np.zeros_like(ref)
    a64, b64, v64 = a.astype(np.float64), b.astype(np.float64), val.astype(np.float64)
    for s in range(n_seg):
        for lo in range(int(seg[s]), int(seg[s + 1]), 1 << 16):
            hi = min(lo + (1 << 16), int(seg[s + 1]))
            x, y = a64[ia[lo:hi]] * v64[lo:hi, None], b64[ib[lo:hi]]
            ref[s] += (x.T @ y).ravel()
            scale[s] += (np.abs(x).T @ np.abs(y)).ravel()
    return ref, scale


def _reduce_cap_len(eng):
    """one segment longer than 2 * num_sms * 1024 nnz: pb200_ttm_reduce caps its blocks and rounds rows per block to 32."""
    return 2 * torch.cuda.get_device_properties(eng.device).multi_processor_count * 1024 + 77


@pytest.mark.parametrize("n_seg", [1, 5, 4096])
@pytest.mark.parametrize("ra,rb", [(5, 6), (60, 60), (64, 65), (70, 24), (130, 40)])
def test_ttm_reduce_matches_f64(eng, ra, rb, n_seg):
    """1x1 up to 3x1 and 2x2 grids of 64x64 output tiles; one segment past the block cap, a few segments with empty ones
    between, 4096 short segments (the limit) with ~30 % empty."""
    rng = np.random.default_rng(100 + ra + rb + n_seg)
    if n_seg == 1:
        lengths = np.array([_reduce_cap_len(eng)])
    elif n_seg == 5:
        lengths = np.array([0, 1, 70_001, 0, 4097])
    else:
        lengths = rng.integers(1, 40, size=n_seg)
        lengths[rng.random(n_seg) < 0.3] = 0
        lengths[[0, -1]] = 0
    seg = np.r_[0, np.cumsum(lengths)].astype(np.int64)
    nnz = int(seg[-1])
    na, nb = 2500, 1800
    ia, ib = rng.integers(0, na, nnz).astype(np.int32), rng.integers(0, nb, nnz).astype(np.int32)
    val = rng.integers(1, 6, size=nnz).astype(np.float32)
    a = rng.uniform(-0.5, 1.0, size=(na, ra)).astype(np.float32)
    b = rng.uniform(-0.5, 1.0, size=(nb, rb)).astype(np.float32)
    args = (n_seg, eng.upload(seg), eng.upload(ia), eng.upload(ib), eng.upload(val), eng.upload(a), ra, eng.upload(b), rb)
    out = eng.ttm_reduce(*args)
    got = out.cpu().numpy().astype(np.float64)
    ref, scale = _xgram_ref(seg, ia, ib, val, a, b)
    assert not got[lengths == 0].any()
    bound = 2.0 ** -22 * (scale + np.abs(ref))
    assert (np.abs(got - ref) <= bound).all(), np.max(np.abs(got - ref) / np.maximum(bound, 1e-300))
    assert torch.equal(out, eng.ttm_reduce(*args))


def test_ttm_reduce_accumulates_in_fp64(eng):
    """One segment of ~1e6 nnz whose terms are all equal and positive (val = 1 as in CoFFee's 0/1 tensor; every factor row
    is the same).  Terms and their sums are exact in fp64, so the kernel must come within the final rounding to fp32.  The
    host repeats the kernel's blocking with an fp32 sum per block (each term val*a*b is exact in fp32: 11-bit mantissas)
    and shows that such a kernel would miss the same bound: equal terms round the same way at every step."""
    rng = np.random.default_rng(5)
    ra, rb, nnz = 5, 6, 1_000_003
    a_row = (rng.integers(1024, 2048, size=ra) / 2048.0).astype(np.float32)
    b_row = (rng.integers(1024, 2048, size=rb) / 2048.0).astype(np.float32)
    na, nb = 700, 900
    a, b = np.tile(a_row, (na, 1)), np.tile(b_row, (nb, 1))
    ia, ib = rng.integers(0, na, nnz).astype(np.int32), rng.integers(0, nb, nnz).astype(np.int32)
    val = np.ones(nnz, dtype=np.float32)
    term = np.outer(a_row.astype(np.float64), b_row.astype(np.float64))
    assert np.array_equal(term.astype(np.float32).astype(np.float64), term)
    ref = (nnz * term).ravel()                                           # exact
    bound = 2.0 ** -22 * (ref + np.abs(ref))                             # scale == ref: all terms positive
    # the kernel's blocking (pb200_ttm_reduce): ceil(len/1024) blocks capped at 2 * num_sms, rows per block rounded to 32
    max_blk = 2 * torch.cuda.get_device_properties(eng.device).multi_processor_count
    nblk = min(-(-nnz // 1024), max_blk)
    rpb = -(-(-(-nnz // nblk)) // 32) * 32
    fp32_blocks = [np.cumsum(np.broadcast_to(term.astype(np.float32), (min(rpb, nnz - lo), ra, rb)), axis=0,
                             dtype=np.float32)[-1].astype(np.float64) for lo in range(0, nnz, rpb)]
    fp32_total = np.sum(fp32_blocks, axis=0).astype(np.float32).astype(np.float64).ravel()
    assert np.max(np.abs(fp32_total - ref) / bound) > 10, "the data no longer tells fp64 from fp32 accumulation"
    seg = eng.upload(np.array([0, nnz], dtype=np.int64))
    out = eng.ttm_reduce(1, seg, eng.upload(ia), eng.upload(ib), eng.upload(val), eng.upload(a), ra, eng.upload(b), rb)
    got = out.cpu().numpy().astype(np.float64).ravel()
    assert (np.abs(got - ref) <= bound).all(), np.max(np.abs(got - ref) / bound)


def test_ttm_reduce_rejects_bad_segments(eng):
    nnz = 10
    z32 = eng.upload(np.zeros(nnz, dtype=np.int32))
    val = eng.upload(np.ones(nnz, dtype=np.float32))
    f = eng.upload(np.ones((1, 3), dtype=np.float32))

    def call(n_seg, seg):
        return eng.ttm_reduce(n_seg, eng.upload(np.asarray(seg, dtype=np.int64)), z32, z32, val, f, 3, f, 3)

    with pytest.raises(ValueError):
        call(0, [0])
    with pytest.raises(ValueError):
        call(4097, np.r_[np.zeros(4097, dtype=np.int64), nnz])
    with pytest.raises(ValueError):
        call(2, [0, 4, nnz - 1])                     # seg_ptr does not end at nnz
    # all-ones factors: every entry of a segment's output is its length
    np.testing.assert_array_equal(call(2, [0, 4, nnz]).cpu().numpy(), np.repeat([[4.0], [6.0]], 9, axis=1))


# ---------------------------------------------------------------------------------------------------------------------
#  pb200_coo_group
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nnz", [0, 100_000])
@pytest.mark.parametrize("n_keys", [1, 2, 1024, 1025])
def test_coo_group_is_the_stable_argsort(eng, n_keys, nnz):
    """Grouping = numpy's stable argsort of the key, exactly: keys with gaps (empty segments, the first key among them when
    there is more than one), the last key n_keys - 1 always present, n_keys on and just past a power of two."""
    rng = np.random.default_rng(n_keys)
    present = np.flatnonzero(rng.random(n_keys) < 0.5)
    present = np.union1d(present[present > 0], [n_keys - 1])
    key = rng.choice(present, size=nnz).astype(np.int32)
    a = rng.integers(0, 1 << 31, size=nnz, dtype=np.int64).astype(np.int32)
    b = rng.integers(0, 1 << 31, size=nnz, dtype=np.int64).astype(np.int32)
    val = rng.standard_normal(nnz).astype(np.float32)
    seg, ao, bo, vo = eng.coo_group(eng.upload(key), n_keys, eng.upload(a), eng.upload(b), eng.upload(val))
    perm = np.argsort(key, kind="stable")
    np.testing.assert_array_equal(seg.cpu().numpy(), np.r_[0, np.cumsum(np.bincount(key, minlength=n_keys))])
    np.testing.assert_array_equal(ao.cpu().numpy(), a[perm])
    np.testing.assert_array_equal(bo.cpu().numpy(), b[perm])
    np.testing.assert_array_equal(vo.cpu().numpy(), val[perm])


# ---------------------------------------------------------------------------------------------------------------------
#  pb200_tall_svd on the buffers HOOI passes it
# ---------------------------------------------------------------------------------------------------------------------
def _ttm_shaped(rng, n, c):
    """[n x c] float32 matrix with a decaying spectrum, stored in the first c columns of an [n x round_up(c, 4)] buffer
    (the layout of a TTM output) whose padding columns hold NaN: any read of them poisons the result."""
    from polara_b200.engine import round_up
    m = (rng.standard_normal((n, c)) * 0.95 ** np.arange(c)).astype(np.float32)
    buf = np.full((n, round_up(c, 4)), np.nan, dtype=np.float32)
    buf[:, :c] = m
    return m, buf


@pytest.mark.parametrize("n,c,rank", [(5000, 70, 24), (3000, 130, 40), (4000, 261, 40), (3000, 5, 4)])
def test_tall_svd_of_column_slices(eng, n, c, rank):
    """The column slices of _hooi_device (ldm = round_up(c, 4) > c; c >= 160 takes the multi-CTA Jacobi): same sigma, U and
    V^T bits as a contiguous copy, sigma against numpy in f64, U orthonormal."""
    from polara_b200.engine import round_up
    rng = np.random.default_rng(c)
    m, buf = _ttm_shaped(rng, n, c)
    sliced = eng.upload(buf)[:, :c]
    assert sliced.stride(0) == round_up(c, 4) > c
    u, s, vt = eng.tall_svd(sliced, rank, want_vt=True)
    u2, s2, vt2 = eng.tall_svd(eng.upload(m), rank, want_vt=True)
    assert torch.equal(s, s2) and torch.equal(u, u2) and torch.equal(vt, vt2)
    np.testing.assert_allclose(s.cpu().numpy(), np.linalg.svd(m.astype(np.float64), compute_uv=False)[:rank], rtol=1e-6)
    uu = u[:, :rank].cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(uu.T @ uu, np.eye(rank), atol=5e-5)
    assert not u[:, rank:].any()


def test_tall_svd_row_sharded_through_the_reduce_hook(eng):
    """The user-sharded mode-0 step in one process: this rank holds the row block A of M = [A; B] and the reduce hook adds
    the other rank's Gram matrix B^T B (f64) to the buffer it is handed.  sigma must be that of M, and U (A's rows of the
    left singular vectors) the corresponding rows of the unsharded result."""
    rng = np.random.default_rng(9)
    n, c, rank, split = 6000, 70, 24, 3500
    m, buf = _ttm_shaped(rng, n, c)
    full = eng.upload(buf)[:, :c]
    u_full, s_full, vt_full = eng.tall_svd(full, rank, want_vt=True)
    b64 = m[split:].astype(np.float64)
    btb = torch.from_numpy(b64.T @ b64).to(eng.device).reshape(-1)
    seen = []

    def add_other_rank(t):
        assert t.dtype == torch.float64 and t.numel() == c * c
        seen.append(t.numel())
        t += btb

    eng.set_reduce_hook(add_other_rank)
    try:
        u_a, s_a, vt_a = eng.tall_svd(full[:split], rank, want_vt=True)
    finally:
        eng.set_reduce_hook(None)
    assert seen == [c * c]
    s_full, s_a = s_full.cpu().numpy(), s_a.cpu().numpy()
    np.testing.assert_allclose(s_a, s_full, rtol=1e-6)
    # rank-r projection of A's rows, sign free: U_A diag(s) V^T against the same rows of the unsharded factorisation
    proj_a = (u_a[:, :rank].cpu().numpy().astype(np.float64) * s_a) @ vt_a.cpu().numpy()
    proj = (u_full[:split, :rank].cpu().numpy().astype(np.float64) * s_full) @ vt_full.cpu().numpy()
    assert np.abs(proj_a - proj).max() < 1e-5 * s_full[0]


# ---------------------------------------------------------------------------------------------------------------------
#  one HOOI build against an f64 HOOI from the same start
# ---------------------------------------------------------------------------------------------------------------------
def _hooi_f64(idx, val, shape, mlrank, init, iters):
    """float64 HOOI as ``po.hooi`` (lib/tensor.py:37-96, same mode order) from ``init``, with dense SVDs of the unfoldings
    so that the gap after each mode's rank is known.  Returns the factors, the core-norm trace and the smallest
    sigma_r / sigma_{r+1} met on the way."""
    r0, r1, r2 = mlrank
    u1, u2 = (np.asarray(x, dtype=np.float64) for x in init)
    trace, gap = [], np.inf

    def lead(unf, r):
        nonlocal gap
        uu, ss, _ = np.linalg.svd(unf, full_matrices=False)
        if r < len(ss):
            gap = min(gap, ss[r - 1] / ss[r])
        return uu[:, :r], ss[:r]

    for _ in range(iters):
        u0, _ = lead(po.ttm3d(idx, val, shape, u2, u1, 0, 2, 1).reshape(shape[0], -1), r0)
        u1, _ = lead(po.ttm3d(idx, val, shape, u2, u0, 1, 2, 0).reshape(shape[1], -1), r1)
        u2, ss = lead(po.ttm3d(idx, val, shape, u1, u0, 2, 1, 0).reshape(shape[2], -1), r2)
        trace.append(float(np.linalg.norm(ss)))
    return (u0, u1, u2), np.asarray(trace), gap


def _planted_tensor(mlrank, seed=21):
    """4000 x 3000 x 5 with ~2e5 nnz: a planted part of multilinear rank exactly ``mlrank`` plus 1e5 weaker entries at
    random positions.  The planted part is r1 dense blocks a_i b_j c_k over disjoint item groups; block p uses user group
    p mod r0 (disjoint groups of 40 users) and the two levels {q, q+1 mod 4}, q = (p div r0) mod 4, so no user group has two
    blocks on the same levels and the level vectors span the first 4 levels.  The random entries fill every mode beyond
    the planted rank, well below it: each unfolding has a clear gap after its rank.  (Sparse ratings such as
    synth.planted_ratings have no gap at ranks 70 or 130: their trailing spectrum is a bulk.)"""
    r0, r1, _ = mlrank
    rng = np.random.default_rng(seed)
    shape = (4000, 3000, 5)
    users = rng.permutation(shape[0])[: r0 * 40].reshape(r0, 40)
    per = 100_000 // (r1 * 40 * 2)
    items = rng.permutation(shape[1])[: r1 * per].reshape(r1, per)
    idx, val = [], []
    for p in range(r1):
        q = (p // r0) % 4
        uu, ii, kk = np.meshgrid(users[p % r0], items[p], [q, (q + 1) % 4], indexing="ij")
        idx.append(np.stack([uu.ravel(), ii.ravel(), kk.ravel()], axis=1))
        val.append((rng.uniform(0.5, 1.5, 40)[:, None, None] * rng.uniform(0.5, 1.5, per)[None, :, None]
                    * rng.uniform(0.5, 1.5, 2)[None, None, :]).ravel())
    n_rand = 100_000
    idx.append(np.stack([rng.integers(0, s, n_rand) for s in shape], axis=1))
    val.append(0.3 * rng.uniform(0.5, 1.5, n_rand))
    return np.concatenate(idx), np.concatenate(val), shape


@pytest.mark.parametrize("mlrank", [(24, 70, 4), (40, 130, 4)])
def test_hooi_build_matches_f64_hooi(eng, mlrank):
    """_hooi_device from a fixed start against the f64 HOOI from the same start, three iterations.
    (24, 70, 4): mode-0 width 280 = ttm_window_kernel<16>, ttm_reduce on 2x1 tiles.
    (40, 130, 4): mode-0 width 520 = row-owned ttm_kernel<32>, ttm_reduce on 3x1 tiles.
    Core-norm trace within 1e-4, factor subspaces within 1e-2, a rebuild bit-identical, the row-owned TTM (switch "ldg")
    within the same tolerances."""
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CoffeeModel
    idx, val, shape = _planted_tensor(mlrank)
    val = val.astype(np.float32)                      # both sides start from the same fp32 values and factors
    iters = 3
    rs = np.random.RandomState(4)
    init = tuple(np.linalg.qr(rs.rand(n, r))[0].astype(np.float32) for n, r in ((shape[1], mlrank[1]), (shape[2], mlrank[2])))
    ref, ref_trace, gap = _hooi_f64(idx, val, shape, mlrank, init, iters)
    assert gap >= 1.05, "the planted tensor has too small a spectral gap for a subspace comparison: %.4f" % gap
    model = B200CoffeeModel(ArrayData(idx, val, shape, n_feedback=shape[2]))
    model.num_iters, model.growth_tol = iters, -np.inf

    def build():
        u0, u1, u2, core, trace = model._hooi_device(idx, val, shape, mlrank, init=init)
        np.testing.assert_allclose(trace, ref_trace, rtol=1e-4)
        for mode, (got, want) in enumerate(zip((u0, u1, u2), ref)):
            assert subspace_gap(got, want) < 1e-2, mode
        return u0, u1, u2, core, np.asarray(trace)

    first = build()
    second = build()
    for x, y in zip(first, second):
        assert np.array_equal(x, y), "a second build is not bit-identical"
    eng.set_spmm_kernel("ldg")
    try:
        build()
    finally:
        eng.set_spmm_kernel("window")


# ---------------------------------------------------------------------------------------------------------------------
#  CoFFee lists against the model's own factors
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,flat", [("coffee_small", None), ("coffee_flat34", [2, 3])])
def test_coffee_lists_are_valid_topk_of_their_own_factors(golden, name, flat):
    """test_coffee_model_reproduces_reference accepts 95 % agreement with the recorded lists (subspace error of the build);
    a systematic scoring error must not hide in the rest: every list is also a valid top-k (tie-aware, f64) of the CoFFee
    scores (po.coffee_slice_scores) of the model's OWN factors and flattener."""
    import scipy.sparse as sps
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CoffeeModel, flatten_weights
    g = golden(name)
    model = B200CoffeeModel(ArrayData.from_golden(g))
    model.verbose = False
    model.mlrank = tuple(int(x) for x in g["mlrank"])
    model.seed = int(g["seed"])
    model.num_iters = int(g["num_iters"])
    model.growth_tol = float(g["growth_tol"])
    if flat is not None:
        model.flattener = flat
    model.build()
    recs = model.get_recommendations()
    (tu, ti, tf), shape, _ = model._get_test_data()
    f = model.data.fields
    v64 = model.factors[f.itemid].astype(np.float64)
    w64 = model.factors[f.feedback].astype(np.float64)
    s64 = po.coffee_slice_scores(tu, ti, tf, shape[0], v64, w64, model.flattener)
    # E = P V with P[u, i] = w[f] . flatten(w^T) summed over the user's (i, f): fp32 SpMM, then fp32 scores E . V^T
    weight = (w64 @ flatten_weights(w64, model.flattener))[np.asarray(tf, dtype=np.int64)]
    p_abs = sps.csr_matrix((np.abs(weight), (tu, ti)), shape=shape[:2])
    tol = 4e-6 * max(np.asarray(p_abs @ np.abs(v64)).sum(1).max(), 1e-30) * np.abs(v64).max()
    assert check_topk_against_scores(recs, s64, tu, ti, model.topk, tol) > 0.995

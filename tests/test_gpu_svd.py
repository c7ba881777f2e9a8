"""The kernels of the SVD builds (SVDModel.build / ScaledSVD.build -> pb200_rsvd_csr, CoffeeModel.build -> pb200_tall_svd)
against float64 host references computed from the same fp32 inputs, at the shapes where they change code path: the 64-wide
tiles and 32-row steps of the Gram kernels and their cap of 2 * SMs row blocks, the switch from the single-CTA Jacobi
kernel to the per-round one at c = 160, subspaces wider than the matrix, and ranks above the numerical rank.  Also the
format kernels of the same build path: pb200_rescale, pb200_csr_transpose, pb200_coo_to_csr.  H100 only.

Tolerances (DESIGN.md §4).  M is fp32, its Gram matrix G = M^T M is accumulated in fp64 from exact fp32 products, and the
one-sided Jacobi solver works in fp64:
  * eigenvalues: |lam_j - ref_j^2| <= LAM_ERR * sigma_1^2 with LAM_ERR = 2^-40.  The Gram sums have at most ~5000 terms
    per block (n <= 600k rows over <= 264 blocks) plus the block partials: <= 5000 * 2^-53 = 5.6e-13 of |M|^T |M| <=
    sigma_1^2; the Jacobi rotations add O(c * 2^-53) of lam_1.  Hence |sigma_j - ref_j| <= min(LAM_ERR * sigma_1^2 /
    ref_j, sqrt(LAM_ERR) * sigma_1).
  * eigenvectors (rows of V^T): sin of the angle to the reference subspace of a cluster of singular values <= LAM_ERR *
    sigma_1^2 / gap (gap = distance of the cluster's lam to the other lam, Davis-Kahan) + 2^-20 (rounding to fp32).
  * left vectors U = M (v_j / sigma_j), with W = v / sigma rounded to fp32 and an fp32 fmaf chain over c: the rounding of
    W and of the chain puts an error e_j in column j whose component along u_i is about sigma_i * 2^-24 / sigma_j.  So
    |(U^T U - I)_ij| <= U_ORTH(i, j) = 2^-24 * (8 sqrt(c) + 2 (sigma_1 / sigma_i + sigma_1 / sigma_j)): orthonormality
    degrades as sigma_1 / sigma_j grows, which is why singular values at or below TAU * sigma_1 are cut (TAU = 1e-6, the
    SVQB cut of the subspace iteration): their sigma is 0 and their U column exactly zero.  A numpy emulation of the same
    steps (fp64 Gram, eigh, W rounded to fp32, fp32 product) stays below a fifth of U_ORTH at c = 64, 512 and 1024.
  * reconstruction: ||M - U diag(sigma) V^T||_F <= 2^-24 (8 c + 4 sqrt(c)) sigma_1 + ||sigma_ref beyond the kept ones||.
  * pb200_rsvd_csr: Rayleigh-Ritz makes A v_j = sigma_j u_j up to rounding (fp32 SpMM and right multiplies):
    ||A v_j - sigma_j u_j|| <= RITZ_ROUND * sigma_1; ||A^T u_j - sigma_j v_j|| measures convergence of the subspace and is
    bounded per case.
  * every kernel is deterministic: a second run gives the same bits."""
import numpy as np
import pytest
import scipy.sparse as sps
import torch

from oracle import polara_oracle as po

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
LAM_ERR = 2.0 ** -40
TAU = 1e-6                 # sigma_j <= TAU * sigma_1 is cut (csrc/rsvd.cu; the SVQB cut of csrc/dense.cu)
RITZ_ROUND = 2.0 ** -24 * 64


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    return get_engine(0)


# ---------------------------------------------------------------------------------------------------------------------
#  pb200_tall_svd
# ---------------------------------------------------------------------------------------------------------------------
def _orth(rng, n, k):
    q, _ = np.linalg.qr(rng.standard_normal((n, k)))
    return q


def _with_spectrum(rng, n, c, sigma):
    """fp32 [n x c] matrix Q1 diag(sigma) Q2^T (sigma has min(n, c) entries; the singular values of the fp32 matrix differ
    from them by about 2^-24 sigma_1)."""
    k = len(sigma)
    return ((_orth(rng, n, k) * sigma) @ _orth(rng, c, k).T).astype(np.float32)


def _u_orth_bound(c, s1, s):
    r = s1 / s
    return U32 * (8 * np.sqrt(c) + 2 * (r[:, None] + r[None, :]))


def _clusters(ref_s, rel=1e-3):
    """indices of the reference singular values grouped into runs whose neighbours differ by less than ``rel`` relative."""
    groups, cur = [], [0]
    for j in range(1, len(ref_s)):
        if ref_s[j - 1] - ref_s[j] < rel * ref_s[j - 1]:
            cur.append(j)
        else:
            groups.append(cur)
            cur = [j]
    groups.append(cur)
    return groups


def _sin_theta(a, b):
    """sine of the largest principal angle between the column spaces of a and b (b with orthonormal columns), as the norm
    of the part of a's orthonormalised columns outside b's span (accurate for small angles, unlike sqrt(1 - cos^2))."""
    qa, _ = np.linalg.qr(a)
    return float(np.linalg.norm(qa - b @ (b.T @ qa), 2))


def _run_tall_svd(eng, m, rank, ldm=None):
    """pb200_tall_svd on ``m`` stored in the first c columns of an [n x ldm] buffer whose padding holds NaN; run twice,
    the second run must give the same bits.  Returns (u [n x rank], sigma, vt) as float64 numpy arrays."""
    n, c = m.shape
    ldm = c if ldm is None else ldm
    buf = np.full((n, ldm), np.nan, dtype=np.float32)
    buf[:, :c] = m
    d = eng.upload(buf)[:, :c]
    u, s, vt = eng.tall_svd(d, rank, want_vt=True)
    u2, s2, vt2 = eng.tall_svd(d, rank, want_vt=True)
    assert torch.equal(u, u2) and torch.equal(s, s2) and torch.equal(vt, vt2), "pb200_tall_svd is not deterministic"
    assert not u[:, rank:].any(), "padding columns of U must stay zero"
    return (u[:, :rank].cpu().numpy().astype(np.float64), s.cpu().numpy(), vt.cpu().numpy().astype(np.float64))


def _check_cut(s, ref, s1):
    """the cut contract: sigma_j = 0 exactly for the cut columns; never cut above 1e-5 sigma_1, never kept far below TAU."""
    live = s > 0
    assert live[ref >= 1e-5 * s1].all(), "a singular value >= 1e-5 sigma_1 was cut"
    assert (ref[~live] <= 2 * TAU * s1).all(), "cut a singular value above 2 TAU sigma_1"
    assert (ref[live] >= 0.5 * TAU * s1).all(), "kept a singular value below TAU / 2 * sigma_1"
    return live


def _check_sigma(s, ref, s1, live):
    dl = LAM_ERR * s1 * s1
    bound = np.minimum(dl / np.maximum(ref, 1e-300), np.sqrt(dl))
    err = np.abs(s - ref)
    worst = np.argmax(np.where(live, err / bound, 0))
    assert (err[live] <= bound[live]).all(), "sigma_%d = %r, reference %r: |err| = %.3g x bound" % (
        worst, s[worst], ref[worst], err[worst] / bound[worst])


def check_tall_svd(m, u, s, vt, rank):
    """u, s, vt of pb200_tall_svd against np.linalg.svd of the same fp32 matrix in float64 (see the module docstring)."""
    n, c = m.shape
    m64 = m.astype(np.float64)
    ru, rs, rvt = np.linalg.svd(m64, full_matrices=False)
    rs = np.r_[rs, np.zeros(c - len(rs))]                 # n < c: the remaining singular values are zero
    s1 = rs[0]
    assert np.all(np.isfinite(u)) and np.all(np.isfinite(s)) and np.all(np.isfinite(vt))
    live = _check_cut(s, rs[:rank], s1)
    _check_sigma(s, rs[:rank], s1, live)
    assert not u[:, ~live].any(), "U columns of cut singular values must be exact zeros"
    # V^T: rows are fp32 roundings of orthonormal fp64 eigenvectors
    assert np.abs(vt @ vt.T - np.eye(rank)).max() <= 2.0 ** -21
    # U: live columns orthonormal within U_ORTH
    ul, sl = u[:, live], s[live]
    err = np.abs(ul.T @ ul - np.eye(len(sl)))
    bound = _u_orth_bound(c, s1, sl)
    assert (err <= bound).all(), "U^T U - I: %.3g x bound" % (err / bound).max()
    # angles per cluster of reference singular values, for clusters inside the kept columns with a gap to the rest
    lam = rs ** 2
    for g in _clusters(rs):
        if g[-1] >= rank or not live[g].all():
            continue
        others = np.delete(lam, g)
        gap = np.min(np.abs(others[:, None] - lam[g][None, :])) if len(others) else np.inf
        if gap <= 0:
            continue
        dk = LAM_ERR * s1 * s1 / gap
        if dk > 0.1:
            continue
        sin_v = _sin_theta(vt[g].T, rvt[g].T)
        assert sin_v <= dk + 2.0 ** -20, "V cluster %s: sin %.3g, bound %.3g" % (g, sin_v, dk)
        sin_u = _sin_theta(u[:, g], ru[:, g])
        bound_u = dk + U32 * (8 * np.sqrt(c) + 4 * s1 / rs[g[-1]])
        assert sin_u <= bound_u, "U cluster %s: sin %.3g, bound %.3g" % (g, sin_u, bound_u)
    # reconstruction: the kept part against M (what was cut or lies beyond the rank is the allowed residual)
    rec = (u * s) @ vt
    dropped = np.sqrt(np.sum(rs[rank:] ** 2) + np.sum(rs[:rank][~live] ** 2))
    res = np.linalg.norm(m64 - rec)
    bound = U32 * (8 * c + 4 * np.sqrt(c)) * s1 + dropped * (1 + 1e-6)
    assert res <= bound, "||M - U S V^T||_F = %.3g x bound" % (res / bound)


# widths on and around every 64-wide Gram tile edge and the Jacobi switch (159 | 160), with row counts below one 32-row step
# and one past / one short of the 2048-row blocks; some stored with ldm > c and NaN padding
WIDTH_CASES = [
    (17, 1, None), (5, 2, None), (17, 31, 33), (2047, 63, None), (2049, 64, 68), (4095, 65, None), (4097, 127, None),
    (6143, 128, 131), (6145, 129, None), (2049, 159, None), (4097, 160, 161), (2047, 161, None), (3000, 1024, 1028),
]


@pytest.mark.parametrize("n,c,ldm", WIDTH_CASES)
def test_tall_svd_widths_and_row_blocks(eng, n, c, ldm):
    """Geometric spectrum sigma_j = 0.93^j (0.995^j at c = 1024), rank = c.  (17, 31): n < c, the last 14 singular values
    are zero and cut; (3000, 1024): the widest Jacobi problem, which must converge within its sweep budget."""
    rng = np.random.default_rng(n * 7 + c)
    m = _with_spectrum(rng, n, c, (0.93 if c < 1024 else 0.995) ** np.arange(min(n, c)))
    u, s, vt = _run_tall_svd(eng, m, c, ldm)
    check_tall_svd(m, u, s, vt, c)


def test_tall_svd_row_block_cap(eng):
    """n = 600001 rows: the 2 * SMs cap on row blocks makes each block longer than 2048 rows (and not a multiple of 32
    rows short of n), and c = 65 spans two 64-wide tiles with a one-column second tile."""
    n, c = 600_001, 65
    sms = torch.cuda.get_device_properties(eng.device).multi_processor_count
    assert -(-n // (2 * sms)) > 2048
    rng = np.random.default_rng(11)
    m = _with_spectrum(rng, n, c, 0.9 ** np.arange(c))
    u, s, vt = _run_tall_svd(eng, m, 24)
    check_tall_svd(m, u, s, vt, 24)


def _repeated_spectrum(c):
    """clusters of multiplicity 2..8 (exactly equal planned values), separated by a factor 0.7."""
    mult = np.resize([2, 8, 3, 5, 4, 7, 6, 1], c)
    vals = []
    level = 1.0
    for k in mult:
        vals += [level] * int(k)
        level *= 0.7
        if len(vals) >= c:
            break
    return np.asarray(vals[:c])


SPECTRA = {
    "geometric": lambda c: 0.9 ** np.arange(c),
    "repeated": _repeated_spectrum,
    "ladder": lambda c: 10.0 ** -np.linspace(0, 11, c),
    "scaled_up": lambda c: 2.0 ** 60 * 0.9 ** np.arange(c),
    "scaled_down": lambda c: 2.0 ** -60 * 0.9 ** np.arange(c),
}


@pytest.mark.parametrize("c", [12, 96, 200])
@pytest.mark.parametrize("spectrum", sorted(SPECTRA))
def test_tall_svd_spectra(eng, spectrum, c):
    """Repeated singular values (U and V compared by projector onto each cluster), a decade ladder 1 ... 1e-11 (every
    singular value below TAU * sigma_1 cut), values scaled by 2^60 and 2^-60; c = 200 runs the multi-CTA Jacobi kernel."""
    rng = np.random.default_rng(c + len(spectrum))
    m = _with_spectrum(rng, 3001, c, SPECTRA[spectrum](c))
    u, s, vt = _run_tall_svd(eng, m, c, ldm=c + 3)
    check_tall_svd(m, u, s, vt, c)


@pytest.mark.parametrize("n,c,true_rank,rank", [(500, 20, 3, 5), (3000, 64, 4, 12), (4000, 200, 7, 40), (3000, 70, 61, 70)])
def test_tall_svd_rank_above_numerical_rank(eng, n, c, true_rank, rank):
    """Exact low-rank M (an fp32 product of fp32 factors, or c - 61 zero columns in the last case) with more singular
    triplets requested than M has: the columns past the numerical rank come back as sigma = 0 and exact-zero U columns,
    every other U column unit-norm and orthogonal within U_ORTH."""
    rng = np.random.default_rng(true_rank * 100 + rank)
    if true_rank == 61:
        m = rng.standard_normal((n, c)).astype(np.float32)
        m[:, rng.choice(c, c - true_rank, replace=False)] = 0.0
    else:
        a = rng.standard_normal((n, true_rank)).astype(np.float32)
        b = rng.standard_normal((true_rank, c)).astype(np.float32)
        m = (a @ b).astype(np.float32)
    u, s, vt = _run_tall_svd(eng, m, rank)
    assert (s > 0).sum() == true_rank, s
    check_tall_svd(m, u, s, vt, rank)


def test_tall_svd_jacobi_kernels_agree(eng):
    """c = 159 runs the single-CTA Jacobi kernel, the same problem padded by one zero column (c = 160) the per-round
    kernel: the 159 leading singular triplets agree within the f64-Gram bounds, the padding's singular value is cut."""
    rng = np.random.default_rng(159)
    n, c = 4000, 159
    m = _with_spectrum(rng, n, c, 0.96 ** np.arange(c))
    pad = np.zeros((n, c + 1), dtype=np.float32)
    pad[:, :c] = m
    u_a, s_a, vt_a = _run_tall_svd(eng, m, c)
    u_b, s_b, vt_b = _run_tall_svd(eng, pad, c + 1)
    check_tall_svd(pad, u_b, s_b, vt_b, c + 1)
    assert s_b[c] == 0 and not u_b[:, c].any()
    s1 = s_a[0]
    bound = 2 * np.minimum(LAM_ERR * s1 * s1 / s_a, np.sqrt(LAM_ERR) * s1)
    assert (np.abs(s_a - s_b[:c]) <= bound).all()
    assert not vt_b[:c, c].any() or np.abs(vt_b[:c, c]).max() <= 2.0 ** -30
    gaps = np.abs(np.diff(s_a ** 2))
    gap = np.minimum(np.r_[gaps, np.inf], np.r_[np.inf, gaps])
    for j in range(c):
        dk = 2 * LAM_ERR * s1 * s1 / gap[j]
        cos_v = abs(vt_a[j] @ vt_b[j, :c])
        cos_u = abs(u_a[:, j] @ u_b[:, j])
        assert 1 - cos_v <= dk + 2.0 ** -20, j
        assert 1 - cos_u <= dk + U32 * (8 * np.sqrt(c) + 4 * s1 / s_a[j]), j


# ---------------------------------------------------------------------------------------------------------------------
#  pb200_rsvd_csr
# ---------------------------------------------------------------------------------------------------------------------
def _clamped_ell(rank, shape):
    """the subspace width SVDModel.build passes (models.py: default_ell, clamped to the matrix)."""
    from polara_b200.engine import round_up
    from polara_b200.models import default_ell
    ell = default_ell(rank, None)
    return min(ell, round_up(min(shape), 32)) if min(shape) >= 32 else 32


def _upload(eng, a):
    a = sps.csr_matrix(a, dtype=np.float32)
    a.sum_duplicates()
    a.sort_indices()
    a_dev = eng.upload_csr(a.indptr.astype(np.int64), a.indices.astype(np.int32), a.data, a.shape)
    return a, a_dev, eng.transpose(a_dev)


def _run_rsvd(eng, a_dev, at_dev, rank, ell, seed=1, max_iters=8):
    """rank, ell and the iteration budget as SVDModel.build passes them; run twice, same bits."""
    out = eng.rsvd(a_dev, at_dev, rank, ell, max_iters=max_iters, tol=1e-6, seed=seed, want_u=True)
    again = eng.rsvd(a_dev, at_dev, rank, ell, max_iters=max_iters, tol=1e-6, seed=seed, want_u=True)
    for x, y in zip(out[:3], again[:3]):
        assert torch.equal(x, y), "pb200_rsvd_csr is not deterministic"
    v, s, u, _ = out
    assert not v[:, rank:].any() and not u[:, rank:].any(), "padding columns of V / U must stay zero"
    return (v[:, :rank].cpu().numpy().astype(np.float64), s.cpu().numpy(), u[:, :rank].cpu().numpy().astype(np.float64))


def check_rsvd(a, v, s, u, rank, conv_tol):
    """against np.linalg.svd of the dense fp32 matrix in float64: sigma, the two Ritz residuals relative to sigma_1,
    orthonormality of the live columns, the cut contract.  ``conv_tol`` bounds ||A^T u_j - sigma_j v_j|| / sigma_1 and
    |sigma_j - ref_j| / sigma_1 (convergence of the subspace)."""
    a64 = a.toarray().astype(np.float64)
    rs = np.linalg.svd(a64, compute_uv=False)
    rs = np.r_[rs, np.zeros(max(0, rank - len(rs)))]
    s1 = rs[0]
    assert np.isfinite(v).all() and np.isfinite(u).all() and np.isfinite(s).all()
    live = _check_cut(s, rs[:rank], s1)
    assert not u[:, ~live].any(), "U columns of cut singular values must be exact zeros"
    assert (s <= rs[:rank] + RITZ_ROUND * s1).all(), "a Ritz value above the singular value it approximates"
    assert (np.abs(s - rs[:rank]) <= conv_tol * s1 + RITZ_ROUND * s1).all(), np.abs(s - rs[:rank]).max() / s1
    r1 = np.linalg.norm(a64 @ v - u * s, axis=0) / s1
    assert (r1 <= RITZ_ROUND + 2 * TAU * ~live).all(), "||A v - s u|| / s_1 = %.3g" % r1.max()
    r2 = np.linalg.norm(a64.T @ u - v * s, axis=0) / s1
    assert (r2 <= conv_tol + RITZ_ROUND).all(), "||A^T u - s v|| / s_1 = %.3g" % r2.max()
    c = a.shape[1]
    for x in (v, u):
        xl, sl = x[:, live], s[live]
        err = np.abs(xl.T @ xl - np.eye(len(sl)))
        bound = _u_orth_bound(min(c, 1024), s1, sl)
        assert (err <= bound).all(), "orthonormality: %.3g x bound" % (err / bound).max()
    # V columns past the live ones are zero or unit vectors orthogonal to the live ones
    vn = np.linalg.norm(v[:, ~live], axis=0)
    assert ((vn == 0) | (np.abs(vn - 1) <= 1e-3)).all(), vn


def _sparse_random(rng, m, n, density):
    a = sps.random(m, n, density=density, random_state=np.random.RandomState(rng.integers(1 << 30)), format="csr")
    a.data = np.rint(1 + 4 * a.data)
    return a


def _low_rank_sparse(rng, m, n, rank):
    """exact rank-``rank`` sparse matrix: ``rank`` rank-one blocks x y^T on disjoint row and column groups (half the
    rows and columns stay empty)."""
    a = sps.lil_matrix((m, n))
    rows = np.array_split(rng.permutation(m)[: m // 2], rank)
    cols = np.array_split(rng.permutation(n)[: n // 2], rank)
    for k, (r, c) in enumerate(zip(rows, cols)):
        x = rng.integers(1, 4, len(r)).astype(float)
        y = rng.integers(1, 3, len(c)).astype(float)
        a[np.ix_(r, c)] = np.outer(x, y) * (1 + k)
    return a.tocsr()


def _rsvd_matrix(name, rng):
    if name == "tall":
        q = _with_spectrum(rng, 3000, 1000, 0.8 ** np.arange(1000))
        return sps.csr_matrix(q), 10, 64, 1e-6
    if name == "wide":
        q = _with_spectrum(rng, 800, 2500, 0.8 ** np.arange(800))
        return sps.csr_matrix(q), 16, 64, 1e-6
    if name == "narrow_40_rank30":
        return _sparse_random(rng, 5000, 40, 0.3), 30, None, 1e-6
    if name == "narrow_40_rank40":
        return _sparse_random(rng, 5000, 40, 0.3), 40, None, 1e-6
    if name == "narrow_20":
        return _sparse_random(rng, 3000, 20, 0.3), 20, None, 1e-6
    if name == "full_rank_200":
        return _sparse_random(rng, 300, 200, 0.2), 200, 224, 1e-6
    if name == "low_rank":
        return _low_rank_sparse(rng, 2000, 900, 3), 8, 32, 1e-6
    if name == "identical_blocks":
        blk = sps.csr_matrix(_with_spectrum(rng, 200, 100, 0.7 ** np.arange(100)))
        return sps.block_diag([blk] * 4, format="csr"), 12, 64, 1e-6
    if name == "empty_rows_cols":
        a = _sparse_random(rng, 2000, 120, 0.05).tolil()
        a[rng.choice(2000, 600, replace=False), :] = 0
        a[:, rng.choice(120, 40, replace=False)] = 0
        a = a.tocsr()
        a.eliminate_zeros()
        return a, 10, 128, 1e-6
    if name == "single_nonzero":
        return sps.csr_matrix(([3.0], ([123], [45])), shape=(500, 300)), 4, 32, 1e-6
    if name == "heavy_row_col":
        a = _sparse_random(rng, 3000, 150, 0.02).tolil()
        a[17, rng.random(150) < 0.8] = 30.0
        a[rng.random(3000) < 0.9, 149] = 2.0
        return a.tocsr(), 10, 160, 1e-6
    if name == "ell_1024":
        q = _with_spectrum(rng, 3000, 1500, 0.97 ** np.arange(1500))
        return sps.csr_matrix(q), 50, 1024, 1e-6
    raise KeyError(name)


RSVD_CASES = ["tall", "wide", "narrow_40_rank30", "narrow_40_rank40", "narrow_20", "full_rank_200", "low_rank",
              "identical_blocks", "empty_rows_cols", "single_nonzero", "heavy_row_col", "ell_1024"]


@pytest.mark.parametrize("name", RSVD_CASES)
def test_rsvd_matches_dense_svd(eng, name):
    """Tall and wide planted spectra, ell wider than the matrix through the model's clamp (5000 x 40 at ranks 30 and 40,
    3000 x 20), rank = min(shape), an exact rank-3 matrix at rank 8 (the five extra columns are cut), four identical
    blocks (every singular value fourfold), empty rows and columns, a single nonzero, one heavy row and column, ell = 1024.
    Every matrix either has a spectral gap well inside ell or no more columns than ell (the sparse ones with a random
    bulk), so the Ritz values and vectors converge to rounding level."""
    rng = np.random.default_rng(RSVD_CASES.index(name))
    a, rank, ell, conv_tol = _rsvd_matrix(name, rng)
    ell = _clamped_ell(rank, a.shape) if ell is None else ell
    a, a_dev, at_dev = _upload(eng, a)
    v, s, u = _run_rsvd(eng, a_dev, at_dev, rank, ell, max_iters=8 if ell < 1024 else 3)
    check_rsvd(a, v, s, u, rank, conv_tol)


def test_rsvd_single_pass_on_a_subspace_wider_than_the_matrix(eng):
    """max_iters = 0: one pass of the range finder.  With ell >= n_cols the first subspace already is the whole row space,
    so the Rayleigh-Ritz step on it (and not on the Gaussian start) gives the SVD to rounding level."""
    rng = np.random.default_rng(8)
    a, rank, _, conv_tol = _rsvd_matrix("narrow_40_rank30", rng)
    a, a_dev, at_dev = _upload(eng, a)
    v, s, u = _run_rsvd(eng, a_dev, at_dev, rank, _clamped_ell(rank, a.shape), max_iters=0)
    check_rsvd(a, v, s, u, rank, conv_tol)


def test_rsvd_seeds(eng):
    """Two seeds agree within the convergence tolerance; one seed twice gives the same bits (checked by _run_rsvd).  The
    iteration stops once the Ritz values settle to tol = 1e-6; the vectors are then within about sqrt(tol)."""
    rng = np.random.default_rng(3)
    a, rank, ell, conv_tol = _rsvd_matrix("tall", rng)
    a, a_dev, at_dev = _upload(eng, a)
    v1, s1, u1 = _run_rsvd(eng, a_dev, at_dev, rank, ell, seed=1)
    v2, s2, u2 = _run_rsvd(eng, a_dev, at_dev, rank, ell, seed=2)
    assert not np.array_equal(v1, v2)
    np.testing.assert_allclose(s1, s2, rtol=0, atol=(conv_tol + RITZ_ROUND) * s1[0])
    from tests.helpers import subspace_gap
    assert subspace_gap(v1, v2) < 2e-3 and subspace_gap(u1, u2) < 2e-3


def test_rsvd_identity_reduce_hook(eng):
    """World size 1 with an identity reduce hook: same bits as without a hook, and the hook sees, per subspace iteration,
    the f64 Gram matrix of A Q (ell^2) and the f32 panel A^T W (n_cols * ell), then the Rayleigh-Ritz Gram matrix."""
    rng = np.random.default_rng(4)
    a, rank, ell, _ = _rsvd_matrix("narrow_40_rank30", rng)
    ell = _clamped_ell(rank, a.shape)
    a, a_dev, at_dev = _upload(eng, a)
    plain = eng.rsvd(a_dev, at_dev, rank, ell, max_iters=8, tol=1e-6, seed=1, want_u=True)
    seen = []
    eng.set_reduce_hook(lambda t: seen.append((t.dtype, t.numel())))
    try:
        hooked = eng.rsvd(a_dev, at_dev, rank, ell, max_iters=8, tol=1e-6, seed=1, want_u=True)
    finally:
        eng.set_reduce_hook(None)
    for x, y in zip(plain[:3], hooked[:3]):
        assert torch.equal(x, y)
    iters = hooked[3]
    n_cols = a.shape[1]
    assert seen == [(torch.float64, ell * ell), (torch.float32, n_cols * ell)] * (iters + 1) + [(torch.float64, ell * ell)]


# ---------------------------------------------------------------------------------------------------------------------
#  pb200_rescale, pb200_csr_transpose, pb200_coo_to_csr
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rs,cs", [(0.8, 0.4), (1.0, 0.0), (0.5, 1.0), (1.3, 0.0)])
def test_rescale_matches_f64_within_one_ulp(eng, rs, cs):
    """ScaledSVD's scaling against po.scaled_training_matrix in float64: each value within one float32 ulp.  Empty rows
    and columns, rows of more than 32 nnz (several passes of the warp), col_scaling 0 (factor 1 / sqrt(count))."""
    rng = np.random.default_rng(int(rs * 10 + cs * 100))
    a = _sparse_random(rng, 3000, 700, 0.03).tolil()
    a[rng.choice(3000, 300, replace=False), :] = 0
    a[:, rng.choice(700, 70, replace=False)] = 0
    a[5, :] = 0
    a[5, rng.choice(700, 200, replace=False)] = 2.0
    a = sps.csr_matrix(a, dtype=np.float32)
    a.eliminate_zeros()
    a.sort_indices()
    a.data = (a.data * rng.uniform(0.5, 1.5, a.nnz)).astype(np.float32)
    assert np.diff(a.indptr).max() > 32
    a_dev = eng.upload_csr(a.indptr.astype(np.int64), a.indices.astype(np.int32), a.data, a.shape)
    eng.rescale(a_dev, rs, cs)
    got = a_dev.values.cpu().numpy()
    ref = po.scaled_training_matrix(a, rs, cs)
    ref.sort_indices()
    assert np.array_equal(ref.indptr, a.indptr) and np.array_equal(ref.indices, a.indices)
    ulp = np.spacing(np.abs(ref.data).astype(np.float32)).astype(np.float64)
    err = np.abs(got.astype(np.float64) - ref.data)
    assert (err <= ulp).all(), (err / ulp).max()


@pytest.mark.parametrize("n_cols", [1024, 1025, 65536, 65537])
def test_transpose_on_bit_boundaries(eng, n_cols):
    """the transpose sorts on ceil(log2(n_cols)) key bits: n_cols = 2^b and 2^b + 1, with the top columns populated."""
    rng = np.random.default_rng(n_cols)
    m = 700
    a = _sparse_random(rng, m, n_cols, 8.0 / n_cols + 0.002).tolil()
    a[rng.choice(m, 50, replace=False), n_cols - 1] = 7.0
    a[rng.choice(m, 50, replace=False), n_cols // 2] = 6.0
    a = sps.csr_matrix(a, dtype=np.float32)
    a.sort_indices()
    a_dev = eng.upload_csr(a.indptr.astype(np.int64), a.indices.astype(np.int32), a.data, a.shape)
    t = eng.transpose(a_dev)
    ref = a.T.tocsr()
    ref.sort_indices()
    np.testing.assert_array_equal(t.indptr.cpu().numpy(), ref.indptr)
    np.testing.assert_array_equal(t.indices.cpu().numpy(), ref.indices)
    np.testing.assert_array_equal(t.values.cpu().numpy(), ref.data)


@pytest.mark.parametrize("n_rows,n_cols", [(1024, 1024), (17, 61681), (16, 65536), (2, 524289)])
def test_coo_to_csr_on_bit_boundaries(eng, n_rows, n_cols):
    """unsorted triplets with duplicates (the sorting path): the keys row * n_cols + col are sorted on
    ceil(log2(n_rows * n_cols)) bits; n_rows * n_cols = 2^20 and 2^20 + 1 (17 * 61681), 2^20 + 2 (2 * 524289), with the
    largest keys present."""
    rng = np.random.default_rng(n_rows)
    nnz = 60_000
    rows = rng.integers(0, n_rows, nnz)
    cols = rng.integers(0, n_cols, nnz)
    rows[:40], cols[:40] = n_rows - 1, n_cols - 1 - np.arange(40) % 3
    rows[40:80], cols[40:80] = 0, 0
    perm = rng.permutation(nnz)
    rows, cols = rows[perm], cols[perm]
    vals = rng.integers(1, 6, nnz).astype(np.float32)
    got = eng.coo_to_csr(eng.upload(rows), eng.upload(cols), eng.upload(vals), (n_rows, n_cols))
    ref = sps.coo_matrix((vals.astype(np.float64), (rows, cols)), shape=(n_rows, n_cols)).tocsr()
    ref.sum_duplicates()
    ref.sort_indices()
    np.testing.assert_array_equal(got.indptr.cpu().numpy(), ref.indptr)
    np.testing.assert_array_equal(got.indices.cpu().numpy(), ref.indices)
    np.testing.assert_array_equal(got.values.cpu().numpy(), ref.data.astype(np.float32))

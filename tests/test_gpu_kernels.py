"""Per-kernel parity of the CUDA path (through the C-ABI) against the oracle / numpy.
Runs on the H100 only."""
import numpy as np
import pytest
import scipy.sparse as sps
import torch

from oracle import polara_oracle as po
from tests.helpers import check_topk_against_scores, random_seen_csr, subspace_gap

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    return get_engine(0)


def _rand_csr(rng, m, n, density, heavy_col=False):
    a = sps.random(m, n, density=density, random_state=np.random.RandomState(rng.integers(1 << 30)), format="csr",
                   dtype=np.float32)
    a.data = np.rint(1 + 4 * a.data).astype(np.float32)
    if heavy_col:   # one very popular column and one very long row: exercises the block-cooperative path
        col = np.zeros((m, 1), dtype=np.float32); col[rng.random(m) < 0.9] = 2.0
        a = sps.hstack([a[:, :-1], sps.csr_matrix(col)]).tocsr()
        row = np.zeros((1, n), dtype=np.float32); row[0, rng.random(n) < 0.8] = 3.0
        a = sps.vstack([a[:-1], sps.csr_matrix(row)]).tocsr()
    a.sort_indices()
    return a


SPMM_KERNELS = ["ldg", "bulk", "cpasync", "window", "window32"]


@pytest.fixture(params=SPMM_KERNELS)
def spmm_kernel(request, eng):
    eng.set_spmm_kernel(request.param)
    yield request.param
    eng.set_spmm_kernel("window")


@pytest.mark.parametrize("m,n,density,ell,heavy", [(1000, 700, 0.02, 32, False), (6000, 9000, 0.004, 64, True),
                                                   (300, 50, 0.3, 96, False), (5000, 6000, 0.01, 160, True),
                                                   (17, 5, 0.5, 32, False)])
def test_spmm_matches_scipy(eng, spmm_kernel, m, n, density, ell, heavy):
    rng = np.random.default_rng(0)
    a = _rand_csr(rng, m, n, density, heavy)
    x = rng.standard_normal((n, ell)).astype(np.float32)
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
    y = eng.spmm(a_dev, eng.upload(x)).cpu().numpy()
    ref = a.astype(np.float64) @ x.astype(np.float64)
    scale = np.abs(a).astype(np.float64) @ np.abs(x).astype(np.float64) + 1e-6
    assert np.max(np.abs(y - ref) / scale) < 5e-6
    # determinism: bit-identical on a second run
    y2 = eng.spmm(a_dev, eng.upload(x)).cpu().numpy()
    assert np.array_equal(y, y2)


def _rows_csr(lengths, n_cols, rng):
    """CSR with prescribed row lengths (distinct sorted columns per row)."""
    indptr = np.zeros(len(lengths) + 1, dtype=np.int64)
    np.cumsum(lengths, out=indptr[1:])
    idx = np.concatenate([np.sort(rng.choice(n_cols, size=k, replace=False)) for k in lengths] or [np.zeros(0, np.int64)])
    val = rng.integers(1, 6, size=indptr[-1]).astype(np.float32)
    return sps.csr_matrix((val, idx.astype(np.int32), indptr), shape=(len(lengths), n_cols))


@pytest.mark.parametrize("lengths", [
    [0, 0, 2048, 0, 2048, 0, 0],                 # rows ending exactly on window boundaries, empty rows around them
    [5000, 0, 0, 1, 9000, 3, 0],                 # rows straddling several 2048-nnz windows (carried pieces)
    [0] * 70 + [1] + [0] * 70,                   # long runs of empty rows, more than one pointer window of 32 rows
    [2047, 1, 1, 2047, 2, 2046, 4096, 0],        # boundaries one off in both directions
    [0, 0, 0],                                   # empty matrix with rows
    [31, 33, 32, 0, 64, 1] * 40,                 # many short rows, group-sized
])
@pytest.mark.parametrize("ell", [32, 96])
def test_spmm_window_and_carry_edges(eng, spmm_kernel, lengths, ell):
    """The staged kernel splits work by nnz windows of 2048: rows that end on, start on or straddle a window boundary,
    empty rows at every position and rows longer than several windows must all come out exact and deterministic."""
    rng = np.random.default_rng(11)
    n_cols = 12000
    a = _rows_csr(lengths, n_cols, rng)
    x = rng.standard_normal((n_cols, ell)).astype(np.float32)
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
    y = eng.spmm(a_dev, eng.upload(x)).cpu().numpy()
    ref = a.astype(np.float64) @ x.astype(np.float64)
    scale = np.abs(a).astype(np.float64) @ np.abs(x).astype(np.float64) + 1e-6
    assert y.shape == ref.shape and np.isfinite(y).all()
    assert np.max(np.abs(y - ref) / scale) < 5e-6
    assert not y[np.asarray(lengths) == 0].any()          # empty rows are written as zeros (Y starts out as garbage)
    assert np.array_equal(y, eng.spmm(a_dev, eng.upload(x)).cpu().numpy())


@pytest.mark.parametrize("m,n,density,ell,n_panels", [(3000, 5000, 0.01, 96, 4), (500, 7001, 0.02, 64, 7),
                                                        (4000, 900, 0.02, 160, 3), (60, 50, 0.5, 32, 50)])
def test_spmm_panel_major_matches_plain(eng, spmm_kernel, m, n, density, ell, n_panels):
    """pb200_csr_block_columns: panel-major copy (virtual row = panel * n_rows + row, global column ids) and the
    panel-by-panel accumulating product; layout checked against numpy, product against scipy, determinism."""
    rng = np.random.default_rng(12)
    a = _rand_csr(rng, m, n, density, True)
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
    panel_cols = -(-n // n_panels)
    b = eng.block_columns(a_dev, panel_cols)
    assert b.n_panels == -(-n // panel_cols) and b.indptr.shape[0] == b.n_panels * m + 1
    # reference layout: for every panel the sub-matrix of its columns, stacked
    coo = a.tocoo()
    order = np.lexsort((coo.col, coo.row, coo.col // panel_cols))
    np.testing.assert_array_equal(b.indices.cpu().numpy(), coo.col[order])
    np.testing.assert_array_equal(b.values.cpu().numpy(), coo.data[order])
    vrow = (coo.col[order] // panel_cols).astype(np.int64) * m + coo.row[order]
    ref_ptr = np.zeros(b.n_panels * m + 1, dtype=np.int64)
    np.cumsum(np.bincount(vrow, minlength=b.n_panels * m), out=ref_ptr[1:])
    np.testing.assert_array_equal(b.indptr.cpu().numpy(), ref_ptr)
    np.testing.assert_array_equal(np.ctypeslib.as_array(b.panel_ptr), ref_ptr[::m][: b.n_panels + 1] if m else 0)
    x = rng.standard_normal((n, ell)).astype(np.float32)
    y = eng.spmm(b, eng.upload(x)).cpu().numpy()
    ref = a.astype(np.float64) @ x.astype(np.float64)
    scale = np.abs(a).astype(np.float64) @ np.abs(x).astype(np.float64) + 1e-6
    assert np.max(np.abs(y - ref) / scale) < 5e-6
    assert np.array_equal(y, eng.spmm(b, eng.upload(x)).cpu().numpy())


def test_coo_to_csr_matches_scipy(eng):
    """pb200_coo_to_csr vs scipy's coo->csr (models.py:169-174): unsorted triplets with duplicates (summed), the two
    columns of an [nnz x 2] index array (stride 2), float64 values; then the sorted fast path; then zero dropping."""
    rng = np.random.default_rng(13)
    m, n, nnz = 700, 900, 20000
    idx = np.stack([rng.integers(0, m, nnz), rng.integers(0, n, nnz)], axis=1).astype(np.int64)
    idx[:500] = idx[500:1000]                                  # duplicates
    val = rng.integers(1, 6, nnz).astype(np.float64)
    ref = sps.coo_matrix((val, (idx[:, 0], idx[:, 1])), shape=(m, n)).tocsr()
    ref.sum_duplicates(); ref.sort_indices()
    idx_d = eng.upload(idx)
    got = eng.coo_to_csr(idx_d[:, 0], idx_d[:, 1], eng.upload(val), (m, n))
    np.testing.assert_array_equal(got.indptr.cpu().numpy(), ref.indptr)
    np.testing.assert_array_equal(got.indices.cpu().numpy(), ref.indices)
    np.testing.assert_array_equal(got.values.cpu().numpy(), ref.data.astype(np.float32))
    # sorted, duplicate-free input (what test_to_coo of a sorted frame gives): no sort, same answer; float32 values
    coo = ref.tocoo()
    got2 = eng.coo_to_csr(eng.upload(coo.row.astype(np.int64)), eng.upload(coo.col.astype(np.int64)),
                          eng.upload(coo.data.astype(np.float32)), (m, n))
    np.testing.assert_array_equal(got2.indptr.cpu().numpy(), ref.indptr)
    np.testing.assert_array_equal(got2.indices.cpu().numpy(), ref.indices)
    np.testing.assert_array_equal(got2.values.cpu().numpy(), ref.data.astype(np.float32))
    # zero feedback is dropped from the matrix (models.py:197-201) but the pattern call keeps it (vals=None -> ones)
    val0 = coo.data.copy(); val0[::7] = 0.0
    keep = val0 != 0
    ref0 = sps.csr_matrix((val0[keep], (coo.row[keep], coo.col[keep])), shape=(m, n))
    got0 = eng.coo_to_csr(eng.upload(coo.row.astype(np.int64)), eng.upload(coo.col.astype(np.int64)), eng.upload(val0), (m, n),
                          drop_zeros=True)
    np.testing.assert_array_equal(got0.indptr.cpu().numpy(), ref0.indptr)
    np.testing.assert_array_equal(got0.indices.cpu().numpy(), ref0.indices)
    np.testing.assert_array_equal(got0.values.cpu().numpy(), ref0.data.astype(np.float32))
    pat = eng.coo_to_csr(eng.upload(coo.row.astype(np.int64)), eng.upload(coo.col.astype(np.int64)), None, (m, n))
    np.testing.assert_array_equal(pat.indices.cpu().numpy(), ref.indices)
    assert (pat.values.cpu().numpy() == 1).all()
    # empty input and out-of-range indices
    e = eng.coo_to_csr(eng.upload(np.zeros(0, np.int64)), eng.upload(np.zeros(0, np.int64)), None, (5, 4))
    assert e.nnz == 0 and not e.indptr.cpu().numpy().any()
    with pytest.raises(ValueError):
        eng.coo_to_csr(eng.upload(np.array([0, 9], np.int64)), eng.upload(np.array([1, 1], np.int64)), None, (5, 4))


@pytest.mark.parametrize("ell,ldx", [(50, 64), (1, 32), (33, 40), (70, 96), (130, 160)])
def test_spmm_live_columns_only(eng, spmm_kernel, ell, ldx):
    """ell need not be a multiple of 32: X is read up to column ell (the rest may hold anything), Y comes back in whole
    groups of 32 columns with zeros beyond ell, and the live columns are bit-identical to the padded call."""
    rng = np.random.default_rng(5)
    a = _rand_csr(rng, 700, 900, 0.02, True)
    x = rng.standard_normal((900, ldx)).astype(np.float32)
    x_poison = x.copy(); x_poison[:, ell:] = np.nan
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
    y = eng.spmm(a_dev, eng.upload(x_poison), ell=ell).cpu().numpy()
    assert y.shape == (700, (ell + 31) // 32 * 32)
    assert not y[:, ell:].any() and np.isfinite(y).all()
    x_zero = x.copy(); x_zero[:, ell:] = 0
    full = eng.spmm(a_dev, eng.upload(np.ascontiguousarray(np.pad(x_zero, ((0, 0), (0, y.shape[1] + 32 - ldx))))), ell=y.shape[1]).cpu().numpy()
    assert np.array_equal(y[:, :ell], full[:, :ell])


def test_spmm_empty_rows_and_empty_matrix(eng, spmm_kernel):
    a = sps.csr_matrix((np.array([1.0, 2.0], dtype=np.float32), (np.array([3, 3]), np.array([0, 4]))), shape=(9, 5))
    x = np.arange(5 * 32, dtype=np.float32).reshape(5, 32)
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
    y = eng.spmm(a_dev, eng.upload(x)).cpu().numpy()
    np.testing.assert_array_equal(y, (a @ x))
    z = sps.csr_matrix((4, 5), dtype=np.float32)
    z_dev = eng.upload_csr(z.indptr, np.zeros(0, np.int32), np.zeros(0, np.float32), z.shape)
    y = eng.spmm(z_dev, eng.upload(x)).cpu().numpy()
    assert y.shape == (4, 32) and not y.any()


@pytest.mark.parametrize("m,n,density,heavy", [(2000, 1500, 0.01, True), (64, 9000, 0.02, False), (5, 3, 0.6, False)])
def test_transpose_matches_scipy(eng, m, n, density, heavy):
    rng = np.random.default_rng(1)
    a = _rand_csr(rng, m, n, density, heavy)
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
    t = eng.transpose(a_dev)
    ref = a.T.tocsr(); ref.sort_indices()
    np.testing.assert_array_equal(t.indptr.cpu().numpy(), ref.indptr)
    np.testing.assert_array_equal(t.indices.cpu().numpy(), ref.indices)
    np.testing.assert_array_equal(t.values.cpu().numpy(), ref.data)


def test_rescale_matches_oracle(eng, golden):
    g = golden("kernels_small")
    a = sps.csr_matrix((g["a_data"], g["a_indices"], g["a_indptr"]), shape=tuple(g["a_shape"]))
    for rs, cs in ((0.7, 1.0), (1.0, 0.4), (0.8, 0.4)):
        a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
        eng.rescale(a_dev, rs, cs)
        got = sps.csr_matrix((a_dev.values.cpu().numpy(), a.indices, a.indptr), shape=a.shape).toarray()
        ref = po.scaled_training_matrix(a, rs, cs).toarray()
        np.testing.assert_allclose(got, ref, rtol=2e-6)
    # and against the recorded reference outputs
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
    eng.rescale(a_dev, 0.7, 1.0)
    got = sps.csr_matrix((a_dev.values.cpu().numpy(), a.indices, a.indptr), shape=a.shape).toarray()
    np.testing.assert_allclose(got, g["sc_rows"], rtol=2e-6)


@pytest.mark.parametrize("n,c,rank", [(5000, 64, 10), (777, 130, 40), (40, 5, 5), (3600, 5, 3),
                                      (4000, 200, 50), (3000, 333, 20), (2500, 160, 40)])     # c >= 160: multi-CTA Jacobi
def test_tall_svd_matches_numpy(eng, n, c, rank):
    rng = np.random.default_rng(2)
    base = rng.standard_normal((n, c)) * (0.8 ** np.arange(c))
    m = base.astype(np.float32)
    u, s, vt = eng.tall_svd(eng.upload(m), rank, want_vt=True)
    uu, ss, vvt = np.linalg.svd(m.astype(np.float64), full_matrices=False)
    np.testing.assert_allclose(s.cpu().numpy(), ss[:rank], rtol=2e-5)
    u = u[:, :rank].cpu().numpy(); vt = vt.cpu().numpy()
    # compare the rank-`rank` reconstruction (sign/rotation free)
    rec = (u * s.cpu().numpy()) @ vt
    ref = (uu[:, :rank] * ss[:rank]) @ vvt[:rank]
    assert np.abs(rec - ref).max() < 2e-4 * ss[0]
    np.testing.assert_allclose(u.T @ u, np.eye(rank), atol=5e-5)


def _planted(n_users, n_items, per_user, rank, seed):
    from polara_b200.synth import planted_ratings
    u, i, r = planted_ratings(n_users, n_items, per_user, rank=rank, decay=0.75, seed=seed)
    return sps.csr_matrix((r, (u, i)), shape=(n_users, n_items)), (u, i, r)


@pytest.mark.parametrize("rank,ell", [(10, 32), (16, 64)])
def test_rsvd_matches_arpack(eng, rank, ell):
    a, _ = _planted(3000, 1200, 50, 24, seed=3)
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
    at_dev = eng.transpose(a_dev)
    v, sigma, u, iters = eng.rsvd(a_dev, at_dev, rank, ell, max_iters=16, tol=1e-8, seed=1, want_u=True)
    assert eng.last_rsvd_info["iters"] == iters and eng.last_rsvd_info["value_change"] >= 0
    v_ref, s_ref, u_ref = po.svd_build(a, rank, return_u=True)
    np.testing.assert_allclose(sigma.cpu().numpy(), s_ref, rtol=1e-4)
    assert subspace_gap(v[:, :rank].cpu().numpy(), v_ref) < 1e-2
    assert subspace_gap(u[:, :rank].cpu().numpy(), u_ref) < 1e-2
    vv = v[:, :rank].cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(vv.T @ vv, np.eye(rank), atol=1e-4)
    # padding columns of the device buffer stay zero (they are read by the SpMM)
    assert not v[:, rank:].any()


@pytest.mark.parametrize("kernel", ["simt", "tc"])
@pytest.mark.parametrize("m,n,r,k,filt", [(200, 1000, 10, 10, True), (333, 4097, 50, 10, True), (64, 300, 7, 25, True),
                                          (130, 2500, 128, 10, False), (50, 40, 5, 10, True), (1, 513, 16, 3, True)])
def test_score_topk_matches_oracle(eng, kernel, m, n, r, k, filt):
    rng = np.random.default_rng(5)
    eng.set_score_kernel(kernel)
    e = (rng.standard_normal((m, r)) * (0.9 ** np.arange(r))).astype(np.float32)
    v = rng.standard_normal((n, r)).astype(np.float32)
    per_row = rng.integers(0, min(n, 40), size=m)
    if n <= 64:
        per_row[: m // 2] = n - 4           # fewer unseen items than k: seen items must re-enter in score order
    rows, cols, indptr = random_seen_csr(rng, m, n, per_row)
    e_dev, v_dev = eng.upload(e), eng.upload(v)
    seen = (eng.upload(indptr), eng.upload(cols.astype(np.int32))) if filt else None
    ids, sc = eng.score_topk(e_dev, v_dev, r, k, seen=seen, want_scores=True)
    ids, sc = ids.cpu().numpy(), sc.cpu().numpy()
    s64 = e.astype(np.float64) @ v.astype(np.float64).T
    tol = 4e-6 * np.abs(e).astype(np.float64).sum(1).max() * np.abs(v).max()
    frac = check_topk_against_scores(ids, s64, rows if filt else [], cols if filt else [], k, tol)
    assert frac > 0.99
    # reported scores are the canonical fp32 scores of the reported items
    got = np.take_along_axis(s64, ids, axis=1)
    np.testing.assert_allclose(sc, got, atol=tol)


def test_score_kernels_agree_bitwise(eng):
    """The tensor-core kernel (bf16 filter + exact rescoring) must return exactly what the
    exact fp32 SIMT kernel returns: same ids, same scores."""
    rng = np.random.default_rng(6)
    m, n, r, k = 700, 20000, 50, 10
    e = rng.standard_normal((m, r)).astype(np.float32)
    v = rng.standard_normal((n, r)).astype(np.float32)
    rows, cols, indptr = random_seen_csr(rng, m, n, rng.integers(0, 200, size=m))
    e_dev, v_dev = eng.upload(e), eng.upload(v)
    seen = (eng.upload(indptr), eng.upload(cols.astype(np.int32)))
    out = {}
    for kernel in ("simt", "tc"):
        eng.set_score_kernel(kernel)
        ids, sc = eng.score_topk(e_dev, v_dev, r, k, seen=seen, want_scores=True)
        out[kernel] = (ids.cpu().numpy(), sc.cpu().numpy())
    np.testing.assert_array_equal(out["simt"][0], out["tc"][0])
    np.testing.assert_array_equal(out["simt"][1], out["tc"][1])


@pytest.mark.parametrize("k", [1, 10, 32, 33, 40])
def test_score_probe_selection_paths(eng, k):
    """The probe kernel picks each user's k best of the 256 largest-norm items through a threshold + compaction + ranking
    fast path (k <= 32, at most 32 keys at or above the threshold) and falls back to k rounds of warp-wide extraction
    otherwise.  Rows built to hit every branch -- zero embeddings (all scores tie), duplicated item rows (equal scores,
    order by id), users who have seen almost the whole head (fewer than k unseen probe items), k > 32 -- must come out
    exactly as from the exact SIMT kernel."""
    rng = np.random.default_rng(77 + k)
    m, n, r = 300, 1500, 24
    e = rng.standard_normal((m, r)).astype(np.float32)
    v = rng.standard_normal((n, r)).astype(np.float32)
    v[:300] *= 3.0                                         # the head of the norm order
    v[10:40] = v[50:80]                                    # equal scores for different ids, inside the head
    e[::7] = 0.0                                           # every score ties at 0
    e[3::11] = np.round(e[3::11])                          # coarse values: many exact ties
    head = np.argsort(-np.linalg.norm(v.astype(np.float64), axis=1), kind="stable")[:256]
    per = []
    for u in range(m):
        if u % 5 == 0:
            keep = rng.choice(256, size=int(rng.integers(0, 6)), replace=False)       # 0..5 unseen head items
            seen = np.setdiff1d(head, head[keep])
        else:
            seen = rng.choice(n, size=int(rng.integers(0, 60)), replace=False)
        per.append(np.sort(seen))
    indptr = np.zeros(m + 1, dtype=np.int64)
    indptr[1:] = np.cumsum([len(x) for x in per])
    cols = np.concatenate(per).astype(np.int32)
    e_dev, v_dev = eng.upload(e), eng.upload(v)
    seen_dev = (eng.upload(indptr), eng.upload(cols))
    out = {}
    for kernel in ("simt", "tc"):
        eng.set_score_kernel(kernel)
        ids, sc = eng.score_topk(e_dev, v_dev, r, k, seen=seen_dev, want_scores=True)
        out[kernel] = (ids.cpu().numpy(), sc.cpu().numpy())
    eng.set_score_kernel("tc")
    np.testing.assert_array_equal(out["simt"][0], out["tc"][0])
    np.testing.assert_array_equal(out["simt"][1], out["tc"][1])


def test_score_heavy_users_cooperative_flush(eng):
    """Users whose history covers the whole head of the sweep order get no lower bound from the probe pass (fewer than k
    unseen probe items): every item of the following tiles survives the filter until the list holds k entries.  Rows with
    that many survivors are worked off by the whole warp (coop_flush_row); the lists must still equal the exact SIMT
    kernel's bit for bit -- for heavy and ordinary users side by side in one tile."""
    rng = np.random.default_rng(123)
    m, n, r, k = 260, 6000, 16, 10
    e = rng.standard_normal((m, r)).astype(np.float32)
    v = (rng.standard_normal((n, r)) * np.linspace(3.0, 0.3, n)[:, None]).astype(np.float32)
    order = np.argsort(-np.linalg.norm(v.astype(np.float64), axis=1), kind="stable")
    per = []
    for u in range(m):
        if u % 9 == 0:
            seen = order[: 1500 + 10 * u]                  # the head and well beyond: no bound from the probe, long history
        elif u % 9 == 1:
            seen = np.setdiff1d(order[:256], order[rng.choice(256, size=3, replace=False)])   # 3 unseen probe items
        else:
            seen = rng.choice(n, size=int(rng.integers(0, 80)), replace=False)
        per.append(np.sort(seen))
    indptr = np.zeros(m + 1, dtype=np.int64)
    indptr[1:] = np.cumsum([len(x) for x in per])
    cols = np.concatenate(per).astype(np.int32)
    e_dev, v_dev = eng.upload(e), eng.upload(v)
    seen_dev = (eng.upload(indptr), eng.upload(cols))
    out = {}
    for kernel in ("simt", "tc"):
        eng.set_score_kernel(kernel)
        ids, sc = eng.score_topk(e_dev, v_dev, r, k, seen=seen_dev, want_scores=True)
        out[kernel] = (ids.cpu().numpy(), sc.cpu().numpy())
    eng.set_score_kernel("tc")
    np.testing.assert_array_equal(out["simt"][0], out["tc"][0])
    np.testing.assert_array_equal(out["simt"][1], out["tc"][1])
    # and no seen item came back
    for u in range(0, m, 9):
        assert not np.isin(out["tc"][0][u], per[u]).any()


def test_rsvd_reports_convergence_and_panels_change_nothing(eng):
    """pb200_rsvd_csr: (i) the convergence report -- a planted spectrum converges (flag set, both measures under their
    tolerances) well before the cap, a cap of one iteration does not and says so; (ii) panel-major A / A^T give the same
    factors as the plain layout (same products in a different, still fixed, summation order)."""
    a, _ = _planted(3000, 1200, 50, 24, seed=3)
    a_dev = eng.upload_csr(a.indptr, a.indices, a.data, a.shape)
    at_dev = eng.transpose(a_dev)
    v, sigma, _, iters = eng.rsvd(a_dev, at_dev, 10, 64, max_iters=40, tol=1e-6, vec_tol=1e-3, seed=1)
    info = eng.last_rsvd_info
    assert info["converged"] and iters < 40 and info["value_change"] < 1e-6 and info["angle_bound"] <= 1e-3
    eng.rsvd(a_dev, at_dev, 10, 64, max_iters=1, tol=1e-12, vec_tol=1e-9, seed=1)
    assert not eng.last_rsvd_info["converged"] and eng.last_rsvd_info["iters"] == 1
    ab = eng.block_columns(a_dev, 300)
    atb = eng.block_columns(at_dev, 700)
    assert ab.n_panels == 4 and atb.n_panels == 5
    v2, sigma2, _, _ = eng.rsvd(ab, atb, 10, 64, max_iters=40, tol=1e-6, vec_tol=1e-3, seed=1)
    np.testing.assert_allclose(sigma2.cpu().numpy(), sigma.cpu().numpy(), rtol=2e-5)
    assert subspace_gap(v2[:, :10].cpu().numpy(), v[:, :10].cpu().numpy()) < 2e-3


def _score_case(eng, rng, m, n, r, k, scale=1.0, kernel="tc"):
    e = (rng.standard_normal((m, r)) * (0.9 ** np.arange(r)) * scale).astype(np.float32)
    v = rng.standard_normal((n, r)).astype(np.float32)
    rows, cols, indptr = random_seen_csr(rng, m, n, rng.integers(0, min(n, 40), size=m))
    e_dev, v_dev = eng.upload(e), eng.upload(v)
    seen = (eng.upload(indptr), eng.upload(cols.astype(np.int32)))
    out = {}
    for kern in ("simt", kernel):
        eng.set_score_kernel(kern)
        ids, sc = eng.score_topk(e_dev, v_dev, r, k, seen=seen, want_scores=True)
        out[kern] = (ids.cpu().numpy(), sc.cpu().numpy())
    return out


def test_score_tc_ignores_stale_shared_memory(eng):
    """A launch must not pick up the k-th-score exchange entries a previous launch left in shared memory: run a problem
    with 100x larger scores first (its thresholds would wipe out every candidate of the second one), then a different
    problem with single-tile work items, and compare with the exact kernel."""
    rng = np.random.default_rng(21)
    _score_case(eng, rng, 333, 4097, 50, 10, scale=100.0)
    out = _score_case(eng, rng, 333, 4097, 50, 10)
    np.testing.assert_array_equal(out["simt"][0], out["tc"][0])
    np.testing.assert_array_equal(out["simt"][1], out["tc"][1])


@pytest.mark.parametrize("case", ["skewed", "negative", "zero_norm_tail", "few_unseen", "flat"])
def test_score_early_termination_is_exact(eng, case):
    """pb200_set_prune: cutting a user tile's sweep where ||e||*||v|| < seeded k-th score must not change a single id or
    score (bit equality with the full sweep and with the exact SIMT kernel), whatever the sign of the scores; on skewed
    norms it must actually cut (counter [5] grows by less than [6])."""
    rng = np.random.default_rng(31)
    m, n, r, k = 600, 30000, 50, 10
    v = rng.standard_normal((n, r)).astype(np.float32)
    e = rng.standard_normal((m, r)).astype(np.float32)
    per_row = rng.integers(0, 60, size=m)
    if case == "skewed":
        v *= (1.0 / np.arange(1, n + 1) ** 0.8).astype(np.float32)[rng.permutation(n), None]
    elif case == "negative":
        v = -np.abs(v); e = np.abs(e)                       # every score negative: thresholds < 0, nothing may be cut
    elif case == "zero_norm_tail":
        v = np.abs(v) * (1.0 / np.arange(1, n + 1) ** 0.8).astype(np.float32)[:, None]
        v[n // 2:] = 0.0                                    # exact zeros score 0 ...
        e[: m // 2] = -np.abs(e[: m // 2])                  # ... and must beat these users' all-negative other scores
    elif case == "few_unseen":
        n = 600; v = v[:n] * (1.0 / np.arange(1, n + 1)).astype(np.float32)[:, None]
        per_row = np.full(m, n - 4)                         # k > unseen: thresholds stay -inf, seen items re-enter
    rows, cols, indptr = random_seen_csr(rng, m, n, per_row)
    e_dev, v_dev = eng.upload(e), eng.upload(v)
    seen = (eng.upload(indptr), eng.upload(cols.astype(np.int32)))
    out = {}
    for name, kernel, prune in (("simt", "simt", True), ("full", "tc", False), ("cut", "tc", True)):
        eng.set_score_kernel(kernel)
        eng.set_prune(prune)
        s0 = eng.stats()
        ids, sc = eng.score_topk(e_dev, v_dev, r, k, seen=seen, want_scores=True)
        s1 = eng.stats()
        out[name] = (ids.cpu().numpy(), sc.cpu().numpy(), s1[5] - s0[5], s1[6] - s0[6])
    eng.set_prune(True)
    for name in ("full", "cut"):
        np.testing.assert_array_equal(out["simt"][0], out[name][0])
        np.testing.assert_array_equal(out["simt"][1], out[name][1])
    assert out["full"][2] == out["full"][3] > 0              # the full sweep executes every tile product
    if case == "skewed":
        assert out["cut"][2] < 0.5 * out["cut"][3]
    if case == "negative":
        assert out["cut"][2] == out["cut"][3]


def test_score_topk_sharded_merge_equals_unsharded(eng):
    rng = np.random.default_rng(7)
    m, n, r, k = 300, 6000, 32, 10
    e = rng.standard_normal((m, r)).astype(np.float32)
    v = rng.standard_normal((n, r)).astype(np.float32)
    rows, cols, indptr = random_seen_csr(rng, m, n, rng.integers(0, 60, size=m))
    e_dev, v_dev = eng.upload(e), eng.upload(v)
    seen = (eng.upload(indptr), eng.upload(cols.astype(np.int32)))
    full = eng.score_topk(e_dev, v_dev, r, k, seen=seen).cpu().numpy()
    parts = []
    bounds = [0, 1500, 3100, 6000]
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        # seen ids stay global: the kernel compares local id + item_offset
        parts.append(eng.score_topk_cands(e_dev, eng.upload(v[lo:hi]), r, k, seen=seen, item_offset=lo))
    stacked = torch.stack(parts).contiguous()
    merged = eng.merge_cands(stacked, len(parts), m, k).cpu().numpy()
    np.testing.assert_array_equal(merged, full)


def test_score_shards_share_their_bounds_through_the_hook(eng):
    """pb200_set_bound_hook: between probe and sweep every shard's per-user lower bounds are replaced by the maximum over the
    shards.  Emulated in one process: a first round records each shard's own bounds, a second round hands every shard the
    elementwise maximum.  The merged lists must equal the unsharded ones bit for bit, the bounds can only rise, and shards
    of low-norm items must sweep less than before (counter [5] = tile products executed)."""
    rng = np.random.default_rng(17)
    m, n, r, k = 700, 24000, 32, 10
    e = rng.standard_normal((m, r)).astype(np.float32)
    # item norms fall with the id: the last shards hold nothing that can beat the first shard's bounds
    v = (rng.standard_normal((n, r)) * np.geomspace(4.0, 0.05, n)[:, None]).astype(np.float32)
    rows, cols, indptr = random_seen_csr(rng, m, n, rng.integers(0, 60, size=m))
    e_dev, v_dev = eng.upload(e), eng.upload(v)
    seen = (eng.upload(indptr), eng.upload(cols.astype(np.int32)))
    eng.set_score_kernel("tc")
    full = eng.score_topk(e_dev, v_dev, r, k, seen=seen).cpu().numpy()
    bounds = [0, 8000, 16000, 24000]
    shards = [(lo, hi, eng.upload(v[lo:hi])) for lo, hi in zip(bounds[:-1], bounds[1:])]
    own = []

    def swept():
        return eng.stats()[5]

    s0 = swept()
    for lo, hi, v_s in shards:
        eng.score_topk_cands(e_dev, v_s, r, k, seen=seen, item_offset=lo, bound_max=lambda t: own.append(t.clone()))
    swept_alone = swept() - s0
    assert len(own) == len(shards) and all(o.shape == (m,) for o in own)
    best = torch.stack(own).max(dim=0).values

    def share(t):
        assert bool((best >= t).all())
        t.copy_(best)

    s1 = swept()
    parts = [eng.score_topk_cands(e_dev, v_s, r, k, seen=seen, item_offset=lo, bound_max=share) for lo, hi, v_s in shards]
    swept_shared = swept() - s1
    merged = eng.merge_cands(torch.stack(parts).contiguous(), len(parts), m, k).cpu().numpy()
    np.testing.assert_array_equal(merged, full)
    assert swept_shared < swept_alone, (swept_shared, swept_alone)
    # the hook is gone after the call: an ordinary call is not affected
    np.testing.assert_array_equal(eng.score_topk(e_dev, v_dev, r, k, seen=seen).cpu().numpy(), full)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("m,n,k", [(40, 3000, 10), (7, 50, 20), (3, 33, 33), (1, 100000, 5)])
def test_topk_dense_matches_reference_semantics(eng, dtype, m, n, k):
    """pb200_topk_dense / pb200_downvote_dense on a caller's dense block vs the oracle's downvote_seen_items +
    get_topk_elements (models.py:494-519, 522-564): plain top-k, the in-place downvote, and the fused form; including
    rows with fewer than k unseen items (seen ones re-enter in score order)."""
    rng = np.random.default_rng(41)
    s = rng.standard_normal((m, n)).astype(dtype)
    per_row = rng.integers(0, min(n, 30), size=m)
    if n <= 64:
        per_row[:] = n - 3                              # fewer unseen than k
    rows, cols, indptr = random_seen_csr(rng, m, n, per_row)
    s_dev = eng.upload(s)
    # (1) plain top-k == row-wise topsort (scores are tie-free)
    ids = eng.topk_dense(s_dev, k).cpu().numpy()
    np.testing.assert_array_equal(ids, po.get_topk_elements(s.astype(np.float64), k))
    # (2) in-place downvote == the reference formula evaluated in the input dtype, bit for bit; then top-k of the
    # lowered block (the lists: from the float64 formula, which orders the seen items by their original score)
    ref = s.astype(np.float64).copy()
    po.downvote_seen_items(ref, rows, cols)
    exact = s.copy()
    po.downvote_seen_items(exact, rows, cols)
    low = eng.upload(s.copy())
    eng.downvote_dense(low, eng.upload(rows.astype(np.int64)), eng.upload(cols.astype(np.int64)))
    np.testing.assert_array_equal(low.cpu().numpy(), exact)
    ids_low = eng.topk_dense(low, k).cpu().numpy()
    ref_ids = po.get_topk_elements(ref, k)
    np.testing.assert_array_equal(ids_low, ref_ids)
    # (3) fused seen handling gives the same lists without touching the block
    fused, sc = eng.topk_dense(s_dev, k, seen=(eng.upload(indptr), eng.upload(cols.astype(np.int32))), want_scores=True)
    np.testing.assert_array_equal(fused.cpu().numpy(), ref_ids)
    np.testing.assert_array_equal(sc.cpu().numpy(), np.take_along_axis(s, ref_ids, axis=1))
    with pytest.raises(ValueError):
        eng.topk_dense(s_dev, n + 1)


def test_model_surface_topk_and_downvote_hooks(eng):
    """RecommenderModel.get_topk_elements / downvote_seen_items stay callable for foreign dense scores (README.md:48-49
    protocol; models.py:494-564): numpy in, numpy out / in place, results as the reference's."""
    from polara_b200.host import ArrayData
    from polara_b200.models import B200SVDModel
    rng = np.random.default_rng(42)
    m, n = 25, 400
    data = ArrayData(np.zeros((1, 2), dtype=np.int64), np.ones(1), (m, n))
    model = B200SVDModel(data)
    model.topk = 7
    scores = rng.standard_normal((m, n))
    rows, cols, _ = random_seen_csr(rng, m, n, rng.integers(1, 20, size=m))
    ref = scores.copy()
    po.downvote_seen_items(ref, rows, cols)
    mine = scores.copy()
    model.downvote_seen_items(mine, (rows, cols))
    np.testing.assert_allclose(mine, ref, rtol=1e-12)
    np.testing.assert_array_equal(model.get_topk_elements(mine), po.get_topk_elements(ref, 7))
    import scipy.sparse as sps2
    with pytest.raises(NotImplementedError):
        model.get_topk_elements(sps2.csr_matrix(scores))


def test_score_dense_matches_numpy(eng):
    rng = np.random.default_rng(8)
    e = rng.standard_normal((3, 20)).astype(np.float32)
    v = rng.standard_normal((999, 20)).astype(np.float32)
    s = eng.score_dense(eng.upload(e), eng.upload(v), 20).cpu().numpy()
    np.testing.assert_allclose(s, e.astype(np.float64) @ v.astype(np.float64).T, atol=1e-4)


def test_ttm_matches_reference_fixture(eng, golden):
    g = golden("kernels_small")
    idx, val, shp = g["ttm_idx"], g["ttm_val"], tuple(int(s) for s in g["ttm_shape"])
    u, v = g["ttm_u"], g["ttm_v"]      # u: [n1 x 3], v: [n2 x 2] ; fixture = ttm3d_seq(idx,val,shp, v, u, ((2,0),(1,0)))
    i0, i1, i2 = (eng.upload(idx[:, c].astype(np.int32)) for c in range(3))
    vals = eng.upload(val.astype(np.float32))
    seg, a1, a2, vv = eng.coo_group(i0, shp[0], i1, i2, vals)
    out = eng.ttm(shp[0], seg, a2, a1, vv, eng.upload(v.astype(np.float32)), v.shape[1],
                  eng.upload(u.astype(np.float32)), u.shape[1])
    got = out[:, : v.shape[1] * u.shape[1]].cpu().numpy().reshape(shp[0], v.shape[1], u.shape[1])
    np.testing.assert_allclose(got, g["ttm0"], rtol=2e-5, atol=2e-5)
    # few-segment variant: group by mode 2, contract modes 1 and 0
    seg2, b0, b1, vv2 = eng.coo_group(i2, shp[2], i0, i1, vals)
    w0 = np.random.default_rng(0).standard_normal((shp[0], 4)).astype(np.float32)
    red = eng.ttm_reduce(shp[2], seg2, b1, b0, vv2, eng.upload(u.astype(np.float32)), u.shape[1], eng.upload(w0), 4)
    ref = po.ttm3d(idx, val, shp, u, w0.astype(np.float64), 2, 1, 0).reshape(shp[2], -1)
    np.testing.assert_allclose(red.cpu().numpy(), ref, rtol=2e-5, atol=2e-5)


# ---------------------------------------------------------------------------------------------------------------------
#  round-2 parity additions (VERDICT r1, "close the parity gaps")
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r", [61, 62, 64, 128, 189, 190, 200, 333, 500, 600])
def test_score_large_rank_matches_simt_and_oracle(eng, r):
    """Ranks beyond one 128-byte operand atom run the K-slab pipeline of the tensor-core kernel (one 64-wide slab per stage,
    accumulator collects the slabs): 62..509 stay on the tensor cores (counter [6] grows), above that the call falls back
    to the exact CUDA-core kernel.  Either way: bit-identical to the SIMT kernel, valid against f64 scores."""
    rng = np.random.default_rng(50 + r)
    m, n, k = 260, 3000, 10
    e = (rng.standard_normal((m, r)) / np.sqrt(r)).astype(np.float32)
    v = rng.standard_normal((n, r)).astype(np.float32)
    rows, cols, indptr = random_seen_csr(rng, m, n, rng.integers(0, 40, size=m))
    e_dev, v_dev = eng.upload(e), eng.upload(v)
    seen = (eng.upload(indptr), eng.upload(cols.astype(np.int32)))
    eng.set_prune(False)
    try:
        eng.set_score_kernel("simt")
        ids0, sc0 = eng.score_topk(e_dev, v_dev, r, k, seen=seen, want_scores=True)
        eng.set_score_kernel("tc")
        s0 = eng.stats()
        ids1, sc1 = eng.score_topk(e_dev, v_dev, r, k, seen=seen, want_scores=True)
        s1 = eng.stats()
    finally:
        eng.set_prune(True)
    np.testing.assert_array_equal(ids0.cpu().numpy(), ids1.cpu().numpy())
    np.testing.assert_array_equal(sc0.cpu().numpy(), sc1.cpu().numpy())
    on_tensor_cores = (s1[6] - s0[6]) > 0
    assert on_tensor_cores == (r <= 509), "rank %d: tensor-core path %s" % (r, on_tensor_cores)
    s64 = e.astype(np.float64) @ v.astype(np.float64).T
    tol = 4e-6 * np.abs(e).astype(np.float64).sum(1).max() * np.abs(v).max()
    assert check_topk_against_scores(ids1.cpu().numpy(), s64, rows, cols, k, tol) > 0.99


def _worst_case_bf16(rng, shape, exps, sign=1.0):
    """float32 values 2^e * (1 + x), x in [0.875, 1) * 2^-8: the upper seven mantissa bits are zero and the lower sixteen
    sit just under the bf16 tie, so round-to-nearest drops ~2^-8 RELATIVE from every element -- the largest error a bf16
    operand can have -- always in the same direction, while the low bits still make all values distinct."""
    low = rng.integers(0x7000, 0x8000, size=shape).astype(np.uint32)
    bits = ((np.asarray(exps, dtype=np.uint32) + np.uint32(127)) << np.uint32(23)) | low
    out = bits.view(np.float32) * np.float32(1.0)
    return (sign * out).astype(np.float32)


@pytest.mark.parametrize("mode", ["mantissa_one", "random_mantissa"])
@pytest.mark.parametrize("scale_exp", [-10, 0, 10])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_score_filter_adversarial_bf16_rounding(eng, mode, scale_exp, sign):
    """The tensor cores only filter: A = -E and B = V are rounded to bf16 and the margin slot must cover that rounding.
    Worst case by construction (mode mantissa_one): every operand loses the maximal ~2^-8 relative to bf16 rounding, all
    in the same direction, user and item vectors are parallel (no cancellation: s - s~ ~ 2^-7 ||e|| ||v||, the bound
    itself), thousands of items differ only below bf16 resolution (near-ties around every threshold), score magnitudes
    2^-10 .. 2^10, all scores positive or all negative (negative thresholds), a block of users without seen items.
    random_mantissa: the same alignment with arbitrary mantissas.  Lists must stay bit-equal to the exact SIMT kernel,
    with and without the early termination."""
    rng = np.random.default_rng(77)
    m, n, r, k = 384, 6000, 50, 10
    pattern = rng.integers(-3, 4, size=r)                                 # per-dimension magnitude 2^p, shared by E and V
    if mode == "mantissa_one":
        v = _worst_case_bf16(rng, (n, r), pattern[None, :] + np.zeros((n, 1), dtype=np.int64))
        e = _worst_case_bf16(rng, (m, r), pattern[None, :] + scale_exp + np.zeros((m, 1), dtype=np.int64), sign=sign)
    else:
        base = np.exp2(pattern).astype(np.float32)
        v = (base[None, :] * (1.0 + 0.02 * rng.random((n, 1))) * (1.0 + 1e-3 * rng.standard_normal((n, r)))).astype(np.float32)
        e = (sign * np.exp2(scale_exp) * base[None, :] * (1.0 + 0.5 * rng.random((m, 1)))
             * (1.0 + 1e-3 * rng.standard_normal((m, r)))).astype(np.float32)
    per_row = rng.integers(0, 30, size=m)
    per_row[:64] = 0
    rows, cols, indptr = random_seen_csr(rng, m, n, per_row)
    e_dev, v_dev = eng.upload(e), eng.upload(v)
    seen = (eng.upload(indptr), eng.upload(cols.astype(np.int32)))
    res = {}
    for prune in (False, True):
        eng.set_prune(prune)
        for kernel in ("simt", "tc"):
            eng.set_score_kernel(kernel)
            ids, sc = eng.score_topk(e_dev, v_dev, r, k, seen=seen, want_scores=True)
            res[(kernel, prune)] = (ids.cpu().numpy(), sc.cpu().numpy())
    eng.set_prune(True)
    for key in (("tc", False), ("tc", True), ("simt", True)):
        np.testing.assert_array_equal(res[("simt", False)][0], res[key][0])
        np.testing.assert_array_equal(res[("simt", False)][1], res[key][1])


@pytest.mark.parametrize("parts", [9, 16, 33])
def test_merge_many_parts_equals_unsharded(eng, parts):
    """k-way merge with more than 8 lists per user runs the warp kernel (one lane per list): 16 item shards, as on two
    boxes, must give the unsharded lists."""
    rng = np.random.default_rng(60 + parts)
    m, n, r, k = 200, 128 * parts + 77, 24, 10
    e = rng.standard_normal((m, r)).astype(np.float32)
    v = rng.standard_normal((n, r)).astype(np.float32)
    rows, cols, indptr = random_seen_csr(rng, m, n, rng.integers(0, 50, size=m))
    e_dev = eng.upload(e)
    seen = (eng.upload(indptr), eng.upload(cols.astype(np.int32)))
    full = eng.score_topk(e_dev, eng.upload(v), r, k, seen=seen).cpu().numpy()
    bounds = np.linspace(0, n, parts + 1).astype(int)
    lists = [eng.score_topk_cands(e_dev, eng.upload(v[lo:hi]), r, k, seen=seen, item_offset=int(lo))
             for lo, hi in zip(bounds[:-1], bounds[1:])]
    merged = eng.merge_cands(torch.stack(lists).contiguous(), parts, m, k).cpu().numpy()
    np.testing.assert_array_equal(merged, full)


@pytest.mark.parametrize("r,prune", [(200, True), (500, True), (128, False), (500, False)])
def test_score_slab_pipeline_many_tiles(eng, r, prune):
    """K-slab pipeline over hundreds of item tiles and several work items per CTA (the single-issuer rule: a second issuing
    warp would wait on a stage barrier several phases ahead and fall through on a stale one -- seen at C5 scale)."""
    rng = np.random.default_rng(90 + r)
    m, n, k = 132 * 128 * 2 + 77, 40000, 10
    e = (rng.standard_normal((m, r)) / np.sqrt(r)).astype(np.float32)
    v = (rng.standard_normal((n, r)) * (1.0 / np.arange(1, n + 1) ** 0.3)[:, None]).astype(np.float32)
    rows, cols, indptr = random_seen_csr(rng, 512, n, rng.integers(0, 40, size=512))
    indptr = np.concatenate([indptr, np.full(m - 512, indptr[-1])])          # only the first users have seen items
    e_dev, v_dev = eng.upload(e), eng.upload(v)
    seen = (eng.upload(indptr), eng.upload(cols.astype(np.int32)))
    eng.set_prune(prune)
    try:
        eng.set_score_kernel("tc")
        ids1, sc1 = eng.score_topk(e_dev, v_dev, r, k, seen=seen, want_scores=True)
        ids2, sc2 = eng.score_topk(e_dev, v_dev, r, k, seen=seen, want_scores=True)      # run to run
        eng.set_score_kernel("simt")
        sub = slice(0, 4096)
        ids0, sc0 = eng.score_topk(e_dev[sub], v_dev, r, k, seen=(seen[0][:4097], seen[1]), want_scores=True)
    finally:
        eng.set_prune(True); eng.set_score_kernel("tc")
    assert torch.equal(ids1, ids2) and torch.equal(sc1, sc2)
    np.testing.assert_array_equal(ids1[sub].cpu().numpy(), ids0.cpu().numpy())
    np.testing.assert_array_equal(sc1[sub].cpu().numpy(), sc0.cpu().numpy())
    # a sample of rows against f64 scores
    pick = rng.choice(m, 64, replace=False)
    s64 = e[pick].astype(np.float64) @ v.astype(np.float64).T
    got = ids1[pick].cpu().numpy()
    for j, u in enumerate(pick):
        sr = s64[j].copy()
        if u < 512:
            sr[cols[indptr[u]:indptr[u + 1]]] = -np.inf
        ref = np.sort(sr)[::-1][:k]
        np.testing.assert_allclose(s64[j][got[j]], ref, atol=4e-6 * np.abs(e[u]).sum() * np.abs(v).max())

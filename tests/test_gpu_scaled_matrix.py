"""The matrix the scaled models factorise -- the ingest pb200_coo_to_csr followed by pb200_rescale -- and the dense
downvote pb200_downvote_dense, bit for bit against the host emulation of the reference's arithmetic (tests/scaled_exact.py,
itself pinned to the reference by tests/test_oracle_scaling.py).  H100 only.

The feedback holds what a count of stored entries gets wrong: explicit 0.0 and -0.0, duplicate pairs that cancel, a row
and a column made only of zeros.  The reference counts a row's stored entries, zeros included, but its row pass (a sparse
product, also at row_scaling == 1) stores only nonzero results, so a column's count excludes them.  Where the emulation
flags an entry as ambiguous (CUDA's double pow may differ from numpy's by up to 2 ulp), the device may give either
float32 neighbour; everywhere else it must give float32 of the reference's float64 value."""
import numpy as np
import pytest
import scipy.sparse as sps
import torch

from tests import scaled_exact as se
from tests.test_gpu_svd import RITZ_ROUND

pytestmark = pytest.mark.gpu

SCALINGS = [(1, 0.4), (0.8, 0.4), (1.3, 0), (0.5, 1)]


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    return get_engine(0)


def _golden_cases():
    from tests.conftest import load_golden
    return [str(c) for c in load_golden("scaling_cases")["cases"]]


def _bits32(x):
    return np.asarray(x, np.float32).view(np.int32)


def _ingest(eng, idx, val, shape):
    """pb200_coo_to_csr on the two columns of the [nnz x 2] index array (element stride 2), as the models pass them."""
    idx_d = eng.upload(np.ascontiguousarray(idx, dtype=np.int64))
    assert idx_d[:, 0].stride(0) == 2
    return eng.coo_to_csr(idx_d[:, 0], idx_d[:, 1], eng.upload(val), shape)


def check_ingest(a_dev, ref):
    """indptr, indices and values (signed zeros included) equal scipy's coo_matrix(...).tocsr()."""
    np.testing.assert_array_equal(a_dev.indptr.cpu().numpy(), ref.indptr)
    np.testing.assert_array_equal(a_dev.indices.cpu().numpy(), ref.indices)
    got = a_dev.values.cpu().numpy()
    bad = np.flatnonzero(_bits32(got) != _bits32(ref.data))
    assert len(bad) == 0, "ingest values differ at %d entries, first %s: got %r, scipy %r" % (
        len(bad), bad[:5], got[bad[:5]], ref.data[bad[:5]])


def check_scaled(got, ref, rs, cs):
    """``got``: the device's scaled float32 values in the pattern of the unscaled CSR ``ref``.  Entries the reference
    drops are 0.  The others are float32 of the reference value, or either end of the ambiguous range where flagged --
    where the unscaled value is a float32.  The CSR holds float32 before scaling, so float64 feedback (or a float64 sum of
    duplicates) that float32 cannot represent is scaled from its rounded value: there one float32 ulp is allowed (two
    where the factors are ambiguous too)."""
    want, kept, _, _ = se.reference_scaled(ref, rs, cs)
    flag, lo, hi = se.ambiguous(ref, rs, cs)
    assert (got[~kept] == 0).all(), "an entry the reference drops is not zero: %r" % got[~kept][got[~kept] != 0][:5]
    want32 = want.astype(np.float32)
    exact = ref.data.astype(np.float32).astype(np.float64) == ref.data
    ok = (_bits32(got) == _bits32(want32)) | (flag & ((got == lo) | (got == hi)))
    bad = np.flatnonzero(kept & exact & ~ok)
    col_counts = np.bincount(ref.indices[kept], minlength=ref.shape[1])
    assert len(bad) == 0, "%d of %d scaled values differ, first %s: got %r, reference %r (nonzero count of their " \
        "columns %s)" % (len(bad), kept.sum(), bad[:5], got[bad[:5]], want32[bad[:5]], col_counts[ref.indices[bad[:5]]])
    ulp = np.spacing(np.abs(want32)).astype(np.float64)
    err = np.abs(got.astype(np.float64) - want32) / ulp
    inexact = kept & ~exact
    assert (err[inexact] <= np.where(flag, 2, 1)[inexact]).all(), "max error %.3g ulp" % err[inexact].max()
    return exact[kept].mean()


def run_case(eng, idx, val, shape, rs, cs):
    """ingest and rescale; returns the unscaled reference CSR and the share of kept entries checked bit for bit."""
    ref = se.reference_csr(idx, val, shape)
    a_dev = _ingest(eng, idx, val, shape)
    check_ingest(a_dev, ref)
    eng.rescale(a_dev, rs, cs)
    return ref, check_scaled(a_dev.values.cpu().numpy(), ref, rs, cs)


@pytest.mark.parametrize("case", _golden_cases())
def test_ingest_and_rescale_on_recorded_cases(eng, golden, case):
    """the cases the reference was run on (60 x 40 and the 4 x 3 example): f32 and f64 feedback, sorted input (the
    ingest's fast path) and shuffled input with duplicates (its sort path), every (row_scaling, col_scaling) pair."""
    g = golden("scaling_cases")
    p = case + "_"
    idx, val, shape = g[p + "idx"], g[p + "val"], tuple(int(s) for s in g[p + "shape"])
    rs, cs = float(g[p + "row_scaling"]), float(g[p + "col_scaling"])
    ref, exact_share = run_case(eng, idx, val, shape, rs, cs)
    np.testing.assert_array_equal(ref.indptr, g[p + "base_indptr"])
    assert exact_share > (0.1 if case == "f64_inexact" else 0.9)


@pytest.mark.parametrize("rs,cs", SCALINGS)
@pytest.mark.parametrize("kind", ["f32_unsorted", "f32_sorted", "f64_unsorted", "f64_sorted", "f64_inexact"])
def test_ingest_and_rescale_match_emulation(eng, kind, rs, cs):
    """3000 x 500 with rows of up to ~500 entries (many passes of the warp).  f64_inexact: most feedback values (0.3, 0.4,
    ...) are not float32 values; check_scaled holds those to one float32 ulp and the rest to the bit."""
    dtype = np.float32 if kind.startswith("f32") else np.float64
    seed = 100 + 10 * SCALINGS.index((rs, cs)) + ["f32_unsorted", "f32_sorted", "f64_unsorted", "f64_sorted",
                                                  "f64_inexact"].index(kind)
    idx, val = se.feedback_case(seed, 3000, 500, dtype=dtype, sorted_input=kind.endswith("_sorted"),
                                representable=kind != "f64_inexact")
    ref, exact_share = run_case(eng, idx, val, (3000, 500), rs, cs)
    assert np.diff(ref.indptr).max() > 32 and (ref.data == 0).sum() > 1000
    assert exact_share > (0.1 if kind == "f64_inexact" else 0.9)


@pytest.mark.parametrize("rs,cs", [(1, 0.4), (0.8, 0.4)])
def test_row_sharded_column_counts(eng, rs, cs):
    """Two row blocks, each scaled by its own call; the reduce hook adds the other block's nonzero column counts to the
    int32 counts, as an all-reduce over two ranks would.  The blocks together are the unsharded result, bit for bit."""
    shape = (3000, 500)
    idx, val = se.feedback_case(7, *shape)
    whole = _ingest(eng, idx, val, shape)
    eng.rescale(whole, rs, cs)
    h = 1234
    blocks = []
    for lo, hi in ((0, h), (h, shape[0])):
        keep = (idx[:, 0] >= lo) & (idx[:, 0] < hi)
        bidx = idx[keep] - np.array([lo, 0], np.int64)
        blocks.append((_ingest(eng, bidx, val[keep], (hi - lo, shape[1])), hi - lo))
    counts = []
    for b, _ in blocks:
        v = b.values.cpu().numpy()
        counts.append(np.bincount(b.indices.cpu().numpy()[v != 0], minlength=shape[1]).astype(np.int32))
    out, calls = [], []
    for j, (b, _) in enumerate(blocks):
        other = torch.as_tensor(counts[1 - j], device=b.values.device)

        def reduce(t, other=other):
            calls.append((t.dtype, t.numel()))
            t += other
        eng.set_reduce_hook(reduce)
        try:
            eng.rescale(b, rs, cs)
        finally:
            eng.set_reduce_hook(None)
        out.append(b.values.cpu().numpy())
    assert calls == [(torch.int32, shape[1])] * 2
    np.testing.assert_array_equal(np.concatenate([b.indices.cpu().numpy() for b, _ in blocks]),
                                  whole.indices.cpu().numpy())
    assert np.array_equal(_bits32(np.concatenate(out)), _bits32(whole.values.cpu().numpy()))


# ---------------------------------------------------------------------------------------------------------------------
#  model level: the scaled models factorise the reference's scaled matrix
# ---------------------------------------------------------------------------------------------------------------------
RANK = 20          # subspace 64 >= 40 columns: the first subspace is the whole row space, the SVD exact to rounding


def _reference_sigma(g, case):
    p = case + "_scaled_"
    a = sps.csr_matrix((g[p + "data"], g[p + "indices"], g[p + "indptr"]), shape=tuple(g[case + "_shape"]))
    return np.linalg.svd(a.toarray(), compute_uv=False)[:RANK]


def _check_sigma(s, ref):
    """check_rsvd's bound on the singular values (test_gpu_svd.py), with conv_tol = 1e-6."""
    s = np.asarray(s, np.float64)[:RANK]
    err = np.abs(s - ref) / ref[0]
    assert (err <= 1e-6 + RITZ_ROUND).all(), "max |sigma - ref| / sigma_1 = %.3g" % err.max()


def _configure(model, rs, cs):
    model.verbose = False
    model.rank = RANK
    model.row_scaling, model.col_scaling = rs, cs
    return model


@pytest.mark.parametrize("case", ["f32_unsorted_0", "f32_unsorted_1", "f64_unsorted_2", "f32_sorted_3"])
def test_scaled_svd_factorises_the_reference_matrix(golden, case):
    from polara_b200.host import ArrayData
    from polara_b200.models import B200ScaledSVD
    g = golden("scaling_cases")
    p = case + "_"
    data = ArrayData(g[p + "idx"], g[p + "val"], tuple(g[p + "shape"]))
    model = _configure(B200ScaledSVD(data), float(g[p + "row_scaling"]), float(g[p + "col_scaling"]))
    model.build()
    _check_sigma(model.factors["singular_values"], _reference_sigma(g, case))


@pytest.mark.parametrize("precompute", [False, True])
def test_scaled_hybrid_svd_factorises_the_reference_matrix(golden, precompute):
    """identity similarity on both sides: the operator is the scaled matrix itself, formed on the host
    (precompute_auxiliary_matrix) or scaled on the device."""
    from polara_b200.host import ArrayData
    from polara_b200.models import B200ScaledHybridSVD
    g = golden("scaling_cases")
    case = "f32_unsorted_1"
    p = case + "_"
    data = ArrayData(g[p + "idx"], g[p + "val"], tuple(g[p + "shape"]))
    model = _configure(B200ScaledHybridSVD(data), float(g[p + "row_scaling"]), float(g[p + "col_scaling"]))
    model.precompute_auxiliary_matrix = precompute
    model.build()
    _check_sigma(model.factors["singular_values"], _reference_sigma(g, case))


def test_scaled_svd_item_cold_start_factorises_the_reference_matrix(golden):
    from polara_b200.host import ColdStartData
    from polara_b200.models import B200ScaledSVDItemColdStart
    g = golden("scaling_cases")
    case = "f32_unsorted_0"
    p = case + "_"
    shape = tuple(int(s) for s in g[p + "shape"])
    rng = np.random.default_rng(3)
    feats = (rng.random((shape[1], 8)) < 0.4).astype(np.float64)
    feats[np.arange(shape[1]), rng.integers(0, 8, shape[1])] = 1
    cold = (rng.random((4, 8)) < 0.5).astype(np.float64)
    cold[:, 0] = 1
    data = ColdStartData(g[p + "idx"], g[p + "val"], shape, cold_item=[0, 1, 2, 3, 3], cold_user=[0, 5, 9, 2, 4],
                         cold_fdbk=np.ones(5), item_features=feats, cold_item_features=cold)
    model = _configure(B200ScaledSVDItemColdStart(data), float(g[p + "row_scaling"]), float(g[p + "col_scaling"]))
    model.build()
    _check_sigma(model.factors["singular_values"], _reference_sigma(g, case))


# ---------------------------------------------------------------------------------------------------------------------
#  pb200_downvote_dense, pb200_topk_dense
# ---------------------------------------------------------------------------------------------------------------------
def _expected_lists(low, k):
    """(lowered desc, id asc), row by row."""
    ids = np.arange(low.shape[1])
    return np.stack([np.lexsort((ids, -row.astype(np.float64)))[:k] for row in low])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_downvote_matches_reference_chain(eng, dtype):
    """standard-normal scores in an [m x lds] buffer (lds > n, NaN padding), seen pairs with repeats; rows with almost
    every item seen, so the lists reach into the lowered scores.  downvote_dense equals the reference's chain in the
    input dtype bit for bit; topk_dense of the lowered block gives the (lowered desc, id asc) lists.  The fused
    topk_dense(seen=...) path orders seen items by their original score, which the float32 chain can merge into one
    lowered value (a tie the reference leaves unspecified): it is compared on the rows where no such merge happens."""
    rng = np.random.default_rng(11)
    m, n, lds, k = 64, 300, 317, 20
    s = rng.standard_normal((m, n)).astype(dtype)
    per_row = rng.integers(0, 60, m)
    per_row[::4] = n - 5                                       # fewer unseen than k
    rows = np.repeat(np.arange(m), per_row)
    cols = np.concatenate([rng.choice(n, c, replace=False) for c in per_row])
    rep = rng.choice(len(rows), 200, replace=False)
    rows, cols = np.r_[rows, rows[rep]], np.r_[cols, cols[rep]]  # repeated (row, col) pairs
    perm = rng.permutation(len(rows))
    rows, cols = rows[perm].astype(np.int64), cols[perm].astype(np.int64)
    want = se.reference_downvote(s, rows, cols)

    buf = np.full((m, lds), np.nan, dtype=dtype)
    buf[:, :n] = s
    d = eng.upload(buf)
    low = d[:, :n]
    eng.downvote_dense(low, eng.upload(rows), eng.upload(cols))
    got = d.cpu().numpy()
    assert np.isnan(got[:, n:]).all(), "the padding was written"
    got = got[:, :n]
    ib = np.int32 if dtype == np.float32 else np.int64
    bad = np.argwhere(got.view(ib) != want.view(ib))
    assert len(bad) == 0, "%d lowered values differ from the reference chain, first %s: got %r, reference %r" % (
        len(bad), bad[:3].tolist(), got[tuple(bad[:3].T)], want[tuple(bad[:3].T)])

    expected = _expected_lists(want, k)
    np.testing.assert_array_equal(eng.topk_dense(low, k).cpu().numpy(), expected)

    seen = sps.csr_matrix((np.ones(len(rows)), (rows, cols)), shape=(m, n))
    seen.sum_duplicates()
    seen.sort_indices()
    fused = eng.topk_dense(eng.upload(s), k, seen=(eng.upload(seen.indptr.astype(np.int64)),
                                                   eng.upload(seen.indices.astype(np.int32)))).cpu().numpy()
    merged = np.array([len(np.unique(want[u, seen.indices[seen.indptr[u]:seen.indptr[u + 1]]]))
                       != len(np.unique(s[u, seen.indices[seen.indptr[u]:seen.indptr[u + 1]]])) for u in range(m)])
    if dtype == np.float64:
        assert not merged.any()
    assert (~merged[::4]).sum() >= 4, "too few rows without merged seen scores to compare the fused path on"
    np.testing.assert_array_equal(fused[~merged], expected[~merged])

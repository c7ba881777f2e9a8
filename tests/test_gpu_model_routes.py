"""The scoring routes of the device models, pinned bit for bit to explicit engine calls: every source of test data
(torch or numpy CSR, user-sorted triplets), one chunk or streamed, HybridSVD projectors, CoFFee and the rank sweep give
the lists that the ingest (``upload_csr`` / ``coo_to_csr``), the SpMM at the padded width and the fused scoring kernel
give on the same user chunks.  The model's ``score_kernel`` holds for its own call only.  H100 only."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

M_SMALL, M_BIG, N = 3000, 4 * 65536 + 777, 2000
RANK = 12


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    e = get_engine(0)
    e.set_score_kernel("tc")
    yield e
    e.set_score_kernel("tc")


def _csr(m, seed=9):
    from polara_b200.synth import popularity_csr
    return popularity_csr(m, N, 12 * m, seed=seed)


def _data(m, source, seed=9):
    """``ArrayData`` with the test matrix as ``source`` ('torch_csr', 'numpy_csr' or 'triplets'), and its CSR."""
    from polara_b200.host import ArrayData
    indptr, indices, values = _csr(m, seed)
    if source == "triplets":
        user = np.repeat(np.arange(m, dtype=np.int64), np.diff(indptr))
        fdbk = values.astype(np.float64)
        fdbk[::97] = 0.0                                   # zero feedback: out of P, still seen
        return ArrayData(np.zeros((1, 2), dtype=np.int64), np.ones(1), (m, N), user, indices.astype(np.int64), fdbk,
                         (m, N), warm_start=True), (indptr, indices, fdbk)
    data = ArrayData(np.zeros((1, 2), dtype=np.int64), np.ones(1), (m, N))
    csr = (indptr, indices, values)
    if source == "torch_csr":
        csr = tuple(torch.from_numpy(x).pin_memory() for x in csr)
    data.test_csr = (csr, (m, N))
    return data, (indptr, indices, values)


def _model(data, width=RANK, projectors=False, seed=1):
    from polara_b200.models import B200SVDModel
    rng = np.random.default_rng(seed)
    v = np.linalg.qr(rng.standard_normal((N, width)))[0] * (0.9 ** np.arange(width))
    model = B200SVDModel(data)
    model.verbose = False
    model.rank = width
    model.factors = {"userid": None, "itemid": v, "singular_values": np.ones(width)}
    if projectors:
        model.factors["itemid_projector_left"] = v * rng.uniform(0.5, 1.5, (N, 1))
        model.factors["itemid_projector_right"] = v * rng.uniform(0.5, 1.5, (N, 1))
    model._is_ready = True
    return model


def _padded(eng, x):
    """a host factor as the models keep it on the device: float32, zero padded to a multiple of 32 columns."""
    from polara_b200.engine import round_up
    buf = np.zeros((x.shape[0], round_up(x.shape[1], 32)), dtype=np.float32)
    buf[:, :x.shape[1]] = x
    return eng.upload(buf)


def _csr_chunks(eng, csr, bounds):
    indptr, indices, values = csr
    for a, b in zip(bounds[:-1], bounds[1:]):
        lo, hi = int(indptr[a]), int(indptr[b])
        p = eng.upload_csr(indptr[a:b + 1] - lo, indices[lo:hi], values[lo:hi], (b - a, N))
        yield p, (p.indptr, p.indices)


def _triplet_chunks(eng, user, item, vals, bounds, drop_zeros=True):
    """P (zero values dropped unless CoFFee weights) and the pattern of ALL triplets, per chunk of users."""
    cuts = np.searchsorted(user, bounds)
    for a, b, lo, hi in zip(bounds[:-1], bounds[1:], cuts[:-1], cuts[1:]):
        u, i = eng.upload(user[lo:hi] - a), eng.upload(item[lo:hi])
        p = eng.coo_to_csr(u, i, eng.upload(vals[lo:hi]), (b - a, N), drop_zeros=drop_zeros)
        s = eng.coo_to_csr(u, i, None, (b - a, N))
        yield p, (s.indptr, s.indices)


def _chunks(eng, source, csr, bounds):
    if source == "triplets":
        indptr, indices, fdbk = csr
        user = np.repeat(np.arange(len(indptr) - 1, dtype=np.int64), np.diff(indptr))
        return _triplet_chunks(eng, user, indices.astype(np.int64), fdbk, bounds)
    return _csr_chunks(eng, csr, bounds)


def _explicit_lists(eng, chunks, v_fold, v_score, rank, k, filter_seen=True):
    from polara_b200.engine import round_up
    vf, vs = _padded(eng, v_fold), _padded(eng, v_score)
    out = []
    for p, seen in chunks:
        e = eng.spmm(p, vf, ell=round_up(rank, 32))
        out.append(eng.score_topk(e, vs, rank, k, seen=seen if filter_seen else None).cpu().numpy())
    return np.concatenate(out)


def _folds(model):
    f = model.factors
    if "itemid_projector_left" in f:
        return f["itemid_projector_right"], f["itemid_projector_left"]
    return f["itemid"], f["itemid"]


@pytest.mark.parametrize("projectors", [False, True])
@pytest.mark.parametrize("source", ["torch_csr", "numpy_csr", "triplets"])
def test_one_chunk_sources_equal_explicit_calls(eng, source, projectors):
    data, csr = _data(M_SMALL, source)
    model = _model(data, projectors=projectors)
    model.profile_phases = projectors
    recs = model.get_recommendations()
    want = _explicit_lists(eng, _chunks(eng, source, csr, [0, M_SMALL]), *_folds(model), RANK, model.topk)
    assert recs.shape == (M_SMALL, model.topk) and recs.dtype == np.int64
    np.testing.assert_array_equal(recs, want)
    if projectors:
        assert len(model.last_score_timings["chunks"]) == 1


@pytest.mark.parametrize("source", ["torch_csr", "numpy_csr", "triplets"])
def test_streamed_sources_equal_explicit_calls_on_the_same_chunks(eng, source):
    """4 * 65536 + 777 users: a torch CSR and the triplets are cut by stream_schedule, a numpy CSR is one chunk."""
    from polara_b200.models import stream_schedule
    data, csr = _data(M_BIG, source)
    model = _model(data)
    model.profile_phases = True
    recs = model.get_recommendations()
    if source == "numpy_csr":
        bounds = [0, M_BIG]
    else:
        bounds = stream_schedule(M_BIG, torch.cuda.get_device_properties(eng.device).multi_processor_count * 128)
        assert len(bounds) > 2
    assert len(model.last_score_timings["chunks"]) == len(bounds) - 1
    want = _explicit_lists(eng, _chunks(eng, source, csr, bounds), *_folds(model), RANK, model.topk)
    np.testing.assert_array_equal(recs, want)


@pytest.mark.parametrize("kernel", ["tc", "simt"])
def test_coffee_equals_explicit_calls(eng, kernel):
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CoffeeModel, flatten_weights
    rng = np.random.default_rng(4)
    m, n_fb, r1 = 1500, 5, 10
    indptr, indices, _ = _csr(m, seed=4)
    user = np.repeat(np.arange(m, dtype=np.int64), np.diff(indptr))
    item = indices.astype(np.int64)
    level = rng.integers(0, n_fb, len(user)).astype(np.int64)
    data = ArrayData(np.zeros((1, 3), dtype=np.int64), np.ones(1), (m, N, n_fb), user, item, level, (m, N),
                     n_feedback=n_fb)
    model = B200CoffeeModel(data)
    model.verbose = False
    model.score_kernel = kernel
    v = np.linalg.qr(rng.standard_normal((N, r1)))[0]
    w = np.linalg.qr(rng.standard_normal((n_fb, 3)))[0]
    model.factors = {"userid": None, "itemid": v, "rating": w, "core": np.ones((8, r1, 3))}
    model._is_ready = True
    recs = model.get_recommendations()
    assert eng.score_kernel == "tc"
    weights = (w @ flatten_weights(w, model.flattener))[level].astype(np.float32)
    with eng.score_kernel_scope(kernel):
        want = _explicit_lists(eng, _triplet_chunks(eng, user, item, weights, [0, m], drop_zeros=False), v, v, r1,
                               model.topk)
    np.testing.assert_array_equal(recs, want)


@pytest.mark.parametrize("projectors", [False, True])
def test_rank_sweep_at_the_live_rank_equals_get_recommendations(eng, projectors):
    data, _ = _data(M_SMALL, "triplets")
    model = _model(data, width=40, projectors=projectors)
    np.testing.assert_array_equal(model.rank_sweep([40])[40], model.get_recommendations())


def test_rank_sweep_reads_test_csr_as_the_triplets_of_the_same_matrix(eng):
    """rank_sweep reads ``data.test_csr`` when it is set, as get_recommendations does."""
    from polara_b200.host import ArrayData
    data, (indptr, indices, values) = _data(M_SMALL, "torch_csr")
    user = np.repeat(np.arange(M_SMALL, dtype=np.int64), np.diff(indptr))
    triplets = ArrayData(np.zeros((1, 2), dtype=np.int64), np.ones(1), (M_SMALL, N), user, indices.astype(np.int64),
                         values.astype(np.float64), (M_SMALL, N), warm_start=True)
    ranks = [5, 12, 33, 40]
    from_csr = _model(data, width=40).rank_sweep(ranks)
    from_triplets = _model(triplets, width=40).rank_sweep(ranks)
    for r in ranks:
        np.testing.assert_array_equal(from_csr[r], from_triplets[r], err_msg="rank %d" % r)


def test_score_kernel_is_scoped_to_the_call(eng):
    """A model's ``score_kernel`` must not stay on the engine, which every model on the device shares: after a SIMT
    model has scored, a model with ``score_kernel = None`` runs the tensor-core kernel (its tile-product counter,
    ``stats()[5]``, grows)."""
    data, _ = _data(M_SMALL, "triplets")
    simt, default = _model(data), _model(data)
    simt.score_kernel = "simt"
    assert eng.score_kernel == "tc"
    simt.get_recommendations()
    assert eng.score_kernel == "tc"
    simt.rank_sweep([4, RANK])
    assert eng.score_kernel == "tc"
    before = eng.stats()[5]
    default.get_recommendations()
    assert eng.stats()[5] > before
    # restored when the call raises too: pb200_score_topk refuses k > 1024 on the host
    simt.topk = 1025
    with pytest.raises(ValueError, match="k must be in"):
        simt.get_recommendations()
    assert eng.score_kernel == "tc"
    # None keeps whatever the engine has, and leaves it as it was
    eng.set_score_kernel("simt")
    try:
        default.get_recommendations()
        assert eng.score_kernel == "simt"
    finally:
        eng.set_score_kernel("tc")

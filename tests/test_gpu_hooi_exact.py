"""The CoFFee build kernels bit for bit against the host emulation of their summation order (tests/hooi_exact.py,
DESIGN.md §4 "HOOI"), with no tolerance: pb200_ttm on every template instance and row profile under both TTM paths,
pb200_ttm_reduce at every tile grid and segment edge, the products of a real _hooi_device build on the arguments it
passed, and the CoFFee lists against the exact scoring emulation.  Every kernel case runs twice.  H100 only."""
import numpy as np
import pytest
import torch

from tests import hooi_exact as he
from tests.exact_scoring import canonical_scores, expected_lists
from tests.test_gpu_hooi import _planted_tensor

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from polara_b200.engine import get_engine
    return get_engine(0)


@pytest.fixture(params=["window", "ldg"])
def switch(request, eng):
    """the kernel switch: "window" runs the window kernel up to 512 columns, "ldg" the row-owned kernel everywhere"""
    eng.set_spmm_kernel(request.param)
    yield request.param
    eng.set_spmm_kernel("window")


def _kind(switch, width):
    return "window" if switch == "window" and width <= 512 else "ldg"


def _num_sms(eng):
    return torch.cuda.get_device_properties(eng.device).multi_processor_count


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.int32)


def _assert_bits(got, want, what):
    bad = _bits(got) != _bits(want)
    if bad.any():
        at = tuple(np.argwhere(bad)[0])
        raise AssertionError("%s: %d of %d entries differ, first at %s: %r != %r" % (
            what, bad.sum(), bad.size, at, got[at], want[at]))


# ---------------------------------------------------------------------------------------------------------------------
#  pb200_ttm
# ---------------------------------------------------------------------------------------------------------------------
def _ttm_nan(eng, n0, seg, i1, i2, val, u, ru, w, rw):
    """pb200_ttm into an [n0 x ldo] output pre-filled with NaN, ldo = ru*rw + 5"""
    from polara_b200.engine import _p
    ldo = ru * rw + 5
    out = torch.full((n0, ldo), float("nan"), dtype=torch.float32, device=eng.device)
    st = eng.lib.pb200_ttm(eng.h, n0, i1.shape[0], _p(seg, torch.int64), _p(i1, torch.int32), _p(i2, torch.int32),
                           _p(val, torch.float32), _p(u, torch.float32), ru, u.stride(0), _p(w, torch.float32), rw,
                           w.stride(0), _p(out), ldo)
    eng._check(st, "ttm")
    return out.cpu().numpy()


def _check_ttm(eng, switch, lengths, ru, rw, seed):
    """groups the fixture with eng.coo_group as _hooi_device does (it must be the host's stable grouping), runs
    pb200_ttm twice on column slices of the factors (ldu = ru + 3, ldw = rw + 1) and compares bits with the emulation"""
    idx, val, u, w = he.ttm_fixture(lengths, ru, rw, seed)
    n0, width = len(lengths), ru * rw
    key, a, b = (eng.upload(idx[:, c].astype(np.int32)) for c in range(3))
    grouped = eng.coo_group(key, n0, a, b, eng.upload(val))
    host = he.group(idx, val, n0)
    for d, h in zip(grouped, host):
        np.testing.assert_array_equal(d.cpu().numpy(), h)
    u_d, w_d = eng.upload(u)[:, :ru], eng.upload(w)[:, :rw]
    assert u_d.stride(0) == ru + 3 and w_d.stride(0) == rw + 1
    want = he.ttm(_kind(switch, width), *host, u, w, ru, rw)
    for run in range(2):
        got = _ttm_nan(eng, n0, *grouped, u_d, ru, w_d, rw)
        _assert_bits(got[:, :width], want, "run %d" % run)
        assert np.isnan(got[:, width:]).all(), "pb200_ttm wrote past column ru*rw"


@pytest.mark.parametrize("ru,rw", [(3, 2), (5, 24), (4, 32), (3, 43), (4, 60), (4, 64), (3, 86), (4, 128), (5, 103),
                                   (32, 32)])
def test_ttm_widths_bit_exact(eng, switch, ru, rw):
    """ttm_window_kernel<4|8|16> and ttm_kernel<4|8|16|32>, on and just past each width boundary"""
    _check_ttm(eng, switch, he.WIDTH_ROWS, ru, rw, seed=0)


@pytest.mark.parametrize("case", sorted(he.TTM_EDGES))
@pytest.mark.parametrize("ru,rw", [(4, 60), (3, 2)])
def test_ttm_segment_edges_bit_exact(eng, switch, case, ru, rw):
    """rows on and around window, block and long-row boundaries, carried over many windows, empty runs, no nnz at all,
    and the skewed item-like grouping"""
    _check_ttm(eng, switch, he.TTM_EDGES[case], ru, rw, seed=3)


# ---------------------------------------------------------------------------------------------------------------------
#  pb200_ttm_reduce
# ---------------------------------------------------------------------------------------------------------------------
def _reduce_lengths(profile, num_sms):
    if profile == "cap":            # one segment past the block cap (at 114 and at 132 SMs too) between empty ones
        return [0, max(300_001, 2 * num_sms * 1024 + 77), 0]
    if profile == "edges":          # k * 1024 and 32 j +- 1 nnz, empty segments first, last and between
        return [0, 1024, 2048, 3072, 31, 33, 63, 65, 0, 1023, 1025, 32 * 40 - 1, 32 * 40 + 1, 4097, 0]
    rng = np.random.default_rng(4096)  # the segment limit, ~30 % empty
    lengths = rng.integers(1, 13, size=4096)
    lengths[rng.random(4096) < 0.3] = 0
    lengths[[0, -1]] = 0
    return lengths.tolist()


@pytest.mark.parametrize("profile,ra,rb", [("cap", 5, 6), ("cap", 70, 24)] +
                         [(p, ra, rb) for p in ("edges", "many") for ra, rb in ((5, 6), (70, 24), (130, 40), (65, 72))])
def test_ttm_reduce_bit_exact(eng, profile, ra, rb):
    """1x1, 2x1, 3x1 and 2x2 grids of 64 x 64 tiles; the blocking of the device's own SM count"""
    sms = _num_sms(eng)
    lengths = _reduce_lengths(profile, sms)
    seg, ia, ib, val, a, b = he.reduce_fixture(lengths, ra, rb, seed=ra + rb)
    want = he.ttm_reduce(seg, ia, ib, val, a, b, ra, rb, sms)
    args = (len(lengths), eng.upload(seg), eng.upload(ia), eng.upload(ib), eng.upload(val), eng.upload(a), ra,
            eng.upload(b), rb)
    for run in range(2):
        _assert_bits(eng.ttm_reduce(*args).cpu().numpy(), want, "run %d" % run)


# ---------------------------------------------------------------------------------------------------------------------
#  the products of a real build
# ---------------------------------------------------------------------------------------------------------------------
def _record(monkeypatch, eng):
    """wraps Engine.ttm, Engine.ttm_reduce and Engine.tall_svd; every call is downloaded in call order"""
    calls = []
    host = lambda t: t.cpu().numpy()                    # noqa: E731
    ttm, ttm_reduce, tall_svd = eng.ttm, eng.ttm_reduce, eng.tall_svd

    def rec_ttm(n0, seg, i1, i2, val, u, ru, w, rw):
        out = ttm(n0, seg, i1, i2, val, u, ru, w, rw)
        calls.append(("ttm", dict(seg=host(seg), i1=host(i1), i2=host(i2), val=host(val), u=host(u[:, :ru]), ru=ru,
                                  w=host(w[:, :rw]), rw=rw, out=host(out[:, :ru * rw]))))
        return out

    def rec_reduce(n_seg, seg, ia, ib, val, a, ra, b, rb):
        out = ttm_reduce(n_seg, seg, ia, ib, val, a, ra, b, rb)
        calls.append(("reduce", dict(seg=host(seg), ia=host(ia), ib=host(ib), val=host(val), a=host(a[:, :ra]), ra=ra,
                                     b=host(b[:, :rb]), rb=rb, out=host(out))))
        return out

    def rec_svd(m, rank, want_vt=False):
        u, s, vt = tall_svd(m, rank, want_vt=want_vt)
        calls.append(("svd", dict(u=host(u), vt=None if vt is None else host(vt))))
        return u, s, vt

    monkeypatch.setattr(eng, "ttm", rec_ttm)
    monkeypatch.setattr(eng, "ttm_reduce", rec_reduce)
    monkeypatch.setattr(eng, "tall_svd", rec_svd)
    return calls


def _subset(n, k=16):
    return np.unique(np.linspace(0, n - 1, min(n, k)).astype(np.int64))


def _check_ttm_call(c, kind):
    """the recorded output against the emulation on the recorded inputs, in every row and up to 16 factor-W columns"""
    ys = _subset(c["rw"])
    want = he.ttm(kind, c["seg"], c["i1"], c["i2"], c["val"], c["u"], c["w"][:, ys], c["ru"], len(ys))
    got = c["out"].reshape(len(c["seg"]) - 1, c["ru"], c["rw"])[:, :, ys].reshape(want.shape)
    _assert_bits(got, want, "ttm %s %dx%d" % (kind, c["ru"], c["rw"]))


def _check_reduce_call(c, sms):
    """the recorded output against the emulation on the recorded inputs, in up to 16 x 16 (x, y) entries"""
    xs, ys = _subset(c["ra"]), _subset(c["rb"])
    want = he.ttm_reduce(c["seg"], c["ia"], c["ib"], c["val"], c["a"][:, xs], c["b"][:, ys], len(xs), len(ys), sms)
    got = c["out"].reshape(-1, c["ra"], c["rb"])[:, xs][:, :, ys].reshape(want.shape)
    _assert_bits(got, want, "ttm_reduce %dx%d" % (c["ra"], c["rb"]))


def _assert_grouped(c, idx, val, n, mode, others, names):
    want = he.group(idx, val, n, mode, others)
    for name, h in zip(names, want):
        np.testing.assert_array_equal(c[name], h, err_msg="mode %d: %s" % (mode, name))


@pytest.mark.parametrize("mlrank", [(24, 70, 4), (40, 130, 4)])
def test_hooi_build_products_bit_exact(eng, switch, monkeypatch, mlrank):
    """_hooi_device from a fixed start, two iterations, on the planted tensor of test_hooi_build_matches_f64_hooi.
    (24, 70, 4): mode 0 = 4 x 70 columns -> window<16> under "window", mode 1 = 4 x 24 -> window<4>, reduce 70 x 24 =
    2x1 tiles; (40, 130, 4): mode 0 = 4 x 130 -> row-owned ttm_kernel<32> under either switch, mode 1 = 4 x 40 ->
    window<8>, reduce 130 x 40 = 3x1 tiles.  The three products of the first iteration and the mode-0 and mode-2
    products of the second equal the emulation on the inputs they were given, and those inputs are the right ones: the
    grouping of each mode, the factor in each slot (u2 then u1 for mode 0, u2 then u0 for mode 1, u1 then u0 for mode 2)
    and the factors the SVDs before them returned."""
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CoffeeModel
    r0, r1, r2 = mlrank
    idx, val, shape = _planted_tensor(mlrank)
    val = val.astype(np.float32)
    rs = np.random.RandomState(4)
    init = tuple(np.linalg.qr(rs.rand(n, r))[0].astype(np.float32) for n, r in ((shape[1], r1), (shape[2], r2)))
    model = B200CoffeeModel(ArrayData(idx, val, shape, n_feedback=shape[2]))
    model._engine = eng
    model.num_iters, model.growth_tol = 2, -np.inf
    calls = _record(monkeypatch, eng)
    model._hooi_device(idx, val, shape, mlrank, init=init)
    assert [k for k, _ in calls] == ["ttm", "svd", "ttm", "svd", "reduce", "svd"] * 2
    t0, s0, t1, s1, red, s2, t0b, _, _, s1b, redb, _ = (c for _, c in calls)
    sms = _num_sms(eng)
    # iteration 1, mode 0: users, (feedback, item) columns x * r1 + y from (u2, u1)
    _assert_grouped(t0, idx, val, shape[0], 0, (2, 1), ("seg", "i1", "i2", "val"))
    assert (t0["ru"], t0["rw"]) == (r2, r1)
    np.testing.assert_array_equal(t0["u"], init[1])
    np.testing.assert_array_equal(t0["w"], init[0])
    _check_ttm_call(t0, _kind(switch, r2 * r1))
    # mode 1: items, (feedback, user) from (u2, u0)
    _assert_grouped(t1, idx, val, shape[1], 1, (2, 0), ("seg", "i1", "i2", "val"))
    assert (t1["ru"], t1["rw"]) == (r2, r0)
    np.testing.assert_array_equal(t1["u"], init[1])
    np.testing.assert_array_equal(t1["w"], s0["u"][:, :r0])
    _check_ttm_call(t1, _kind(switch, r2 * r0))
    # mode 2: feedback levels, (item, user) from (u1, u0)
    _assert_grouped(red, idx, val, shape[2], 2, (1, 0), ("seg", "ia", "ib", "val"))
    assert (red["ra"], red["rb"]) == (r1, r0)
    np.testing.assert_array_equal(red["a"], s1["u"][:, :r1])
    np.testing.assert_array_equal(red["b"], s0["u"][:, :r0])
    _check_reduce_call(red, sms)
    # iteration 2: mode 0 from the new u2 (the leading rows of the mode-2 V^T) and u1; mode 2 from its own u1 and u0
    np.testing.assert_array_equal(t0b["u"], s2["vt"][:r2].T)
    np.testing.assert_array_equal(t0b["w"], s1["u"][:, :r1])
    _check_ttm_call(t0b, _kind(switch, r2 * r1))
    np.testing.assert_array_equal(redb["a"], s1b["u"][:, :r1])
    _check_reduce_call(redb, sms)


# ---------------------------------------------------------------------------------------------------------------------
#  CoFFee lists
# ---------------------------------------------------------------------------------------------------------------------
_BUILT = {}


def _coffee(golden, name):
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CoffeeModel
    if name not in _BUILT:
        g = golden(name)
        model = B200CoffeeModel(ArrayData.from_golden(g))
        model.verbose = False
        model.mlrank = tuple(int(x) for x in g["mlrank"])
        model.seed = int(g["seed"])
        model.num_iters = int(g["num_iters"])
        model.growth_tol = float(g["growth_tol"])
        model.build()
        _BUILT[name] = model
    return _BUILT[name]


FLATTENERS = {"none": None, "int": 2, "list": [2, 3], "slice": slice(1, 4), "sum": "sum", "mean": "mean",
              "slice_mean": (slice(0, 3), "mean")}


@pytest.mark.parametrize("kernel", ["simt", "tc"])
@pytest.mark.parametrize("flat", sorted(FLATTENERS))
@pytest.mark.parametrize("name", ["coffee_small", "coffee_flat34"])
def test_coffee_lists_bit_exact(golden, monkeypatch, name, flat, kernel):
    """The per-triplet weights the model hands the test matrix are (w . flatten(w^T))[f] cast to fp32; with E = P V
    formed by pb200_spmm on that matrix and the padded item factor, the lists are the exact emulation of the canonical
    scores of E against that factor, seen items filtered."""
    from polara_b200.engine import round_up
    from polara_b200.models import flatten_weights
    model = _coffee(golden, name)
    eng = model.engine
    model.flattener = FLATTENERS[flat]
    model.score_kernel = kernel
    seen_values = []
    test_csr = model._test_csr_device

    def rec(test_data, shape, values=None, **kw):
        seen_values.append(values)
        return test_csr(test_data, shape, values=values, **kw)

    monkeypatch.setattr(model, "_test_csr_device", rec)
    try:
        recs = model.get_recommendations()
    finally:
        model.score_kernel = None
    f = model.data.fields
    (tu, ti, tf), shape, _ = model._get_test_data()
    w = model.factors[f.feedback]
    weights = (w @ flatten_weights(w, FLATTENERS[flat]))[np.asarray(tf, np.int64)].astype(np.float32)
    assert len(seen_values) == 1
    _assert_bits(np.asarray(seen_values[0]), weights, "weights")
    p_dev, seen_dev = test_csr((tu, ti, None), shape, values=weights)
    v_pad = model._device_factor(f.itemid)
    r = model.factors[f.itemid].shape[1]
    e = eng.spmm(p_dev, v_pad, ell=round_up(r, 32))
    seen = (seen_dev[0].cpu().numpy(), seen_dev[1].cpu().numpy()) if model.filter_seen else None
    want, _ = expected_lists(canonical_scores(e.cpu().numpy(), v_pad.cpu().numpy(), r), seen, model.topk)
    np.testing.assert_array_equal(recs, want)

"""CPU-only checks: the C-ABI library loads and exports every declared symbol, host-side
logic (metrics, data replay, rank handling) behaves like the reference."""
import ctypes
import os
import re

import numpy as np
import pytest

from polara_b200 import _abi, _build, host

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    _build.build()
    return _abi.load()


def test_library_exports_every_header_symbol(lib):
    header = open(os.path.join(ROOT, "include", "polara_b200.h")).read()
    declared = set(re.findall(r"\b(pb200_[a-z_0-9]+)\s*\(", header))
    assert declared, "no declarations parsed"
    for name in declared:
        assert hasattr(lib, name), "library does not export %s" % name
    # and the ctypes table binds exactly the declared set
    assert declared == set(_abi.EXPORTED_SYMBOLS)
    assert lib.pb200_version() >= 100


def test_context_creation_fails_loudly_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    handle = ctypes.c_void_p()
    st = lib.pb200_ctx_create(0, None, ctypes.byref(handle))
    assert st != _abi.OK and not handle.value
    from polara_b200.engine import get_engine
    with pytest.raises(RuntimeError):
        get_engine()


def test_product_path_has_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from polara_b200.models import B200SVDModel
    data = host.ArrayData(np.array([[0, 0], [1, 1]]), np.ones(2), (2, 2))
    model = B200SVDModel(data)
    model.verbose = False
    with pytest.raises(RuntimeError):
        model.build()


def test_product_code_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "polara_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith(".py"):
                src = open(os.path.join(dirpath, fn)).read()
                assert "oracle" not in src.replace("no CPU fallback", ""), "%s mentions the oracle" % fn


@pytest.mark.parametrize("name", ["svd_warm_r10", "svd_known_r8", "svd_scaled_r10", "coffee_small"])
def test_evaluate_lists_reproduces_reference_hits(golden, name):
    g = golden(name)
    sp = float(g["switch_positive"]) if "switch_positive" in g else np.nan
    res = host.evaluate_lists(g["recs"], g["holdout_user"], g["holdout_item"], g["holdout_fdbk"],
                              int(g["train_shape"][1]), metric_type="hits",
                              switch_positive=None if np.isnan(sp) else sp)
    ref = g["hits"]
    assert res.true_positive == ref[0] and res.false_negative == ref[3]
    assert float(res.false_positive) == ref[1]
    if ref[2] >= 0:
        assert res.true_negative == ref[2]


def test_evaluate_lists_relevance_recall(golden):
    g = golden("svd_warm_r10")
    rel = host.evaluate_lists(g["recs"], g["holdout_user"], g["holdout_item"], g["holdout_fdbk"],
                              int(g["train_shape"][1]), metric_type="relevance")
    # recall / miss_rate are the well-defined entries of the reference tuple (SURVEY.md §8a A16)
    np.testing.assert_allclose(rel.recall, g["relevance"][1], rtol=1e-12)
    np.testing.assert_allclose(rel.miss_rate, g["relevance"][4], rtol=1e-12)


def test_rank_setter_truncates_like_reference():
    from polara_b200.models import B200SVDModel
    data = host.ArrayData(np.array([[0, 0], [1, 1]]), np.ones(2), (2, 2))
    model = B200SVDModel(data)
    model._rank = 6
    model.factors = {"userid": None, "itemid": np.arange(24.0).reshape(4, 6), "singular_values": np.arange(6.0)}
    model._is_ready = True
    model.rank = 4                                  # models.py:819-832: slice, keep ready
    assert model.factors["itemid"].shape == (4, 4) and model.factors["singular_values"].shape == (4,)
    assert model._is_ready
    model.rank = 5                                  # growing invalidates
    assert not model._is_ready and model.factors["itemid"] is None


def test_build_wrapper_resets_cached_recommendations():
    calls = []

    class M(host.RecommenderModel):
        def build(self):
            calls.append(self._is_ready)

        def get_recommendations(self):
            return np.zeros((1, 1), dtype=np.int64)

    data = host.ArrayData(np.array([[0, 0]]), np.ones(1), (1, 1))
    m = M(data)
    m.verbose = False
    _ = m.recommendations                           # auto-build (models.py:100-108)
    assert calls == [False] and m._is_ready
    m._recommendations = "stale"
    m.build()
    assert m._recommendations is None and m._is_ready


def test_flatten_weights_matches_oracle():
    from oracle import polara_oracle as po
    from polara_b200.models import flatten_weights
    w = np.random.default_rng(0).standard_normal((5, 3))
    for fl in (None, slice(0, None), [2, 3], 1, "sum", (slice(1, 4), "mean")):
        np.testing.assert_allclose(flatten_weights(w, fl), po.flatten_scores(w.T, fl))
    with pytest.raises(NotImplementedError):
        flatten_weights(w, "max")


def test_stream_schedule_covers_users_in_growing_whole_waves():
    """chunk plan of the pinned-CSR fast path: whole waves of the scoring grid, a small first chunk (its upload is the
    only exposed one) and bounded growth so that every later upload hides behind the chunk before it."""
    from polara_b200.models import stream_schedule
    unit = 132 * 128
    for m in (1, 40_000, 250_000, 300_000, 1_000_000, 10_000_000, 12_345_678):
        b = stream_schedule(m, unit)
        assert b[0] == 0 and b[-1] == m and all(x < y for x, y in zip(b[:-1], b[1:]))
        sizes = [y - x for x, y in zip(b[:-1], b[1:])]
        assert all(s % unit == 0 for s in sizes[:-1])                      # only the last chunk may end inside a wave
        if len(sizes) > 1:
            assert sizes[0] <= max(unit, 0.08 * m)
            assert all(nxt <= 1.6 * cur + unit for cur, nxt in zip(sizes[:-2], sizes[1:-1]))
            assert sizes[-1] <= (1.0 + 1.6) * (1.6 * sizes[-2] + unit)


def test_header_is_plain_c_and_links_from_c(tmp_path):
    """The boundary is a C ABI: include/polara_b200.h must compile as C99 and a C program must link against the library
    (no torch, no C++).  Without a GPU the context constructor has to fail with a status code, not crash."""
    import shutil
    import subprocess
    from polara_b200 import _abi
    if shutil.which("gcc") is None or not os.path.exists(_abi.lib_path()):
        pytest.skip("needs gcc and the built library")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "use_abi.c"
    src.write_text('#include <stdio.h>\n#include "polara_b200.h"\n'
                   'int main(void) {\n'
                   '    pb200_ctx* ctx = NULL;\n'
                   '    int v = pb200_version();\n'
                   '    int st = pb200_ctx_create(0, NULL, &ctx);\n'
                   '    printf("%d %d %d\\n", v, st, ctx != NULL);\n'
                   '    if (ctx) pb200_ctx_destroy(ctx);\n'
                   '    return 0;\n}\n')
    exe = tmp_path / "use_abi"
    libdir = os.path.dirname(_abi.lib_path())
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"), str(src), "-o", str(exe),
                    "-L", libdir, "-lpolara_b200", "-Wl,-rpath," + libdir], check=True, capture_output=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    version, status, has_ctx = int(out[0]), int(out[1]), int(out[2])
    assert version == _abi.load().pb200_version()
    import torch
    if not torch.cuda.is_available():
        assert status != 0 and has_ctx == 0
    else:
        assert (status == 0) == (has_ctx == 1)


def test_coffee_mlrank_reduction_rounds_the_core_without_rebuild():
    """CoffeeModel._check_reduced_rank (models.py:949-980): lowering mlrank rotates factors and shrinks the core on the host
    (no rebuild); the rounded model is the best lower-rank approximation inside the old subspaces; raising it invalidates."""
    from oracle import polara_oracle as po
    from polara_b200.models import B200CoffeeModel, round_tucker_core
    rng = np.random.default_rng(4)
    shape, mlrank = (40, 30, 5), (6, 5, 3)
    data = host.ArrayData(np.zeros((1, 3), dtype=np.int64), np.ones(1), shape, n_feedback=5)
    model = B200CoffeeModel(data)
    model.verbose = False
    model._mlrank = mlrank
    f = data.fields
    us = [np.linalg.qr(rng.standard_normal((n, r)))[0] for n, r in zip(shape, mlrank)]
    core = rng.standard_normal(mlrank)
    model.factors = {f.userid: us[0], f.itemid: us[1], f.feedback: us[2], "core": core}
    model._is_ready = True
    backup = model.factors
    model.mlrank = (4, 5, 2)
    assert model._is_ready and model.factors is not backup and backup["core"] is core          # old dict untouched
    want = po.reduce_tucker_rank(us, core, (4, 5, 2))
    for key, ref in zip((f.userid, f.itemid, f.feedback), want[0]):
        np.testing.assert_allclose(model.factors[key], ref, atol=1e-12)
        assert np.abs(model.factors[key].T @ model.factors[key] - np.eye(ref.shape[1])).max() < 1e-12
    np.testing.assert_allclose(model.factors["core"], want[1], atol=1e-12)
    assert model.factors["core"].shape == (4, 5, 2) and model.factors[f.itemid] is us[1]
    # product and oracle agree mode by mode, and a full-rank "reduction" only rotates
    for mode in range(3):
        rot, small = round_tucker_core(core, mode, mlrank[mode])
        rot_o, small_o = po.round_core(core, mode, mlrank[mode])
        np.testing.assert_allclose(rot, rot_o, atol=1e-13)
        np.testing.assert_allclose(small, small_o, atol=1e-13)
        np.testing.assert_allclose(np.tensordot(rot, small, axes=(1, mode)).transpose(np.argsort([mode] + [d for d in range(3) if d != mode])),
                                   core, atol=1e-12)
    model.mlrank = (4, 6, 2)                      # raising a rank cannot be served from the factors
    assert not model._is_ready and model.factors == {}


def test_hook_exception_is_the_cause_of_the_failing_call(monkeypatch):
    """A Python exception raised inside a reduce / bound hook cannot unwind through the C frames: the trampoline parks it,
    the C call comes back with "hook failed", and Engine._check re-raises with the parked exception as the cause."""
    from polara_b200 import _abi, engine

    class Stub(engine.Engine):
        def __init__(self):                       # no device, no context: only the error path is exercised
            self.h = None
            self._reduce_error = ValueError("all_reduce blew up")

    def failing_check(handle, status, where=""):
        raise RuntimeError("polara_b200 %s failed (status %d): bound hook failed with status 1" % (where, status))

    monkeypatch.setattr(_abi, "check", failing_check)
    stub = Stub()
    with pytest.raises(RuntimeError) as info:
        stub._check(4, "score_topk_cands")
    assert isinstance(info.value.__cause__, ValueError) and "all_reduce blew up" in str(info.value.__cause__)
    assert stub._reduce_error is None
    with pytest.raises(RuntimeError) as info:     # nothing parked: the plain error
        stub._check(4, "score_topk_cands")
    assert info.value.__cause__ is None

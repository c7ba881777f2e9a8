"""Generate ``tests/golden/scaling_cases.npz`` by running the REAL reference's scaling of the training matrix on feedback
with explicit zeros, -0.0, duplicates that cancel, a row and a column made only of zeros, empty rows and columns and a
row longer than 32 entries (tests.scaled_exact.feedback_case).  TEST INFRASTRUCTURE; needs the reference checkout named
by POLARA_REFERENCE_ROOT.

    POLARA_REFERENCE_ROOT=... python oracle/make_scaling_golden.py

Stored per case ``<name>_*``: the triplets (``idx``, ``val`` in the feedback dtype), ``shape``, ``row_scaling`` and
``col_scaling``; the unscaled matrix ``SVDModel.get_training_matrix()`` (``base_*``: indptr, indices, data); the row
pass ``rescale_matrix(base, row_scaling, 1)`` (``rows_*``); and ``ScaledSVD.get_training_matrix()`` with those scalings
(``scaled_*``), all read through ``oracle.ref_driver.StubData``.  Also ``dv_*``: float32 and float64 score blocks with
repeated seen pairs and the block ``downvote_seen_items`` leaves (dense branch).
"""
import os
import sys

import numpy as np
import scipy.sparse as sps

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle.ref_driver import StubData  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402
from tests.scaled_exact import feedback_case  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "scaling_cases.npz")
SCALINGS = [(1, 0.4), (0.8, 0.4), (1.3, 0), (0.5, 1)]


def cases():
    """(name, triplets, shape, row_scaling, col_scaling)."""
    shape = (60, 40)
    yield "example", (np.array([(0, 0), (0, 1), (1, 1), (1, 2), (2, 1), (2, 0), (2, 0), (3, 1)], np.int64),
                      np.array([1, 0, 2, 3, 0, 1, -1, 5], np.float64)), (4, 3), 1, 0.4
    for j, (rs, cs) in enumerate(SCALINGS):
        yield "f32_unsorted_%d" % j, feedback_case(10 + j, *shape), shape, rs, cs
        yield "f32_sorted_%d" % j, feedback_case(20 + j, *shape, sorted_input=True), shape, rs, cs
        yield "f64_unsorted_%d" % j, feedback_case(30 + j, *shape, dtype=np.float64), shape, rs, cs
    yield "f64_inexact", feedback_case(40, *shape, dtype=np.float64, representable=False), shape, 1, 0.4


def _csr(res, key, m):
    m = sps.csr_matrix(m)
    m.sort_indices()
    res[key + "_indptr"], res[key + "_indices"] = m.indptr.astype(np.int64), m.indices.astype(np.int64)
    res[key + "_data"] = m.data


def downvote_blocks():
    rng = np.random.default_rng(7)
    for dtype in (np.float32, np.float64):
        m, n = 12, 50
        s = rng.standard_normal((m, n)).astype(dtype)
        rows = rng.integers(0, m, 150)
        cols = rng.integers(0, n, 150)
        rows[-10:], cols[-10:] = rows[:10], cols[:10]                 # repeated pairs
        yield np.dtype(dtype).name, s, rows.astype(np.int64), cols.astype(np.int64)


def main():
    import_reference()
    from polara.preprocessing.matrices import rescale_matrix
    from polara.recommender.models import RecommenderModel, ScaledSVD, SVDModel
    res, names = {}, []
    for name, (idx, val), shape, rs, cs in cases():
        data = StubData(shape, train=(idx, val))
        base = SVDModel(data).get_training_matrix()
        model = ScaledSVD(data)
        model.row_scaling, model.col_scaling = rs, cs
        p = name + "_"
        res.update({p + "idx": idx, p + "val": val, p + "shape": np.array(shape, np.int64),
                    p + "row_scaling": np.array(float(rs)), p + "col_scaling": np.array(float(cs))})
        _csr(res, p + "base", base)
        _csr(res, p + "rows", rescale_matrix(base, rs, 1))
        _csr(res, p + "scaled", model.get_training_matrix())
        names.append(name)
        print("%-16s %s nnz %d stored zeros %d -> %d" % (name, val.dtype, base.nnz, (base.data == 0).sum(),
                                                          res[p + "scaled_data"].size))
    res["cases"] = np.array(names)
    dv = []
    for name, s, rows, cols in downvote_blocks():
        low = s.copy()
        RecommenderModel.downvote_seen_items(low, (rows, cols))
        res.update({"dv_%s_scores" % name: s, "dv_%s_rows" % name: rows, "dv_%s_cols" % name: cols,
                    "dv_%s_lowered" % name: low})
        dv.append(name)
    res["dv_cases"] = np.array(dv)
    np.savez_compressed(OUT, **res)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

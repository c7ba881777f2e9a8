"""CPU checks of the SimilarityAggregation oracle (oracle/sim_oracle.py) against the reference's recorded runs
(tests/golden/sim_cases.npz, made by oracle/make_sim_golden.py), of the item-to-item oracle on the wide catalogue
(tests/golden/i2i_wide_cases.npz), and of the sparse item x item matrix's memory refusal."""
import os

import numpy as np
import pytest
import scipy.sparse as sps

from oracle import i2i_oracle as io
from oracle import sim_oracle as so

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "sim_cases.npz")
WIDE = os.path.join(os.path.dirname(__file__), "golden", "i2i_wide_cases.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN, allow_pickle=False)


def cases():
    return [str(c) for c in np.load(GOLDEN)["cases"]]


def relations(g, c):
    p = c + "_"
    return sps.csr_matrix((g[p + "rel_data"], g[p + "rel_indices"], g[p + "rel_indptr"]), shape=tuple(g[p + "rel_shape"]))


def case_args(g, c):
    p = c + "_"
    return dict(relations=relations(g, c), test_user=g[p + "test_user"], test_item=g[p + "test_item"],
                test_fdbk=g[p + "test_fdbk"], test_shape=tuple(g[p + "test_shape"]), topk=int(g[p + "topk"]),
                filter_seen=bool(g[p + "filter_seen"]), implicit=bool(g[p + "implicit"]),
                dense_output=bool(g[p + "dense_output"]), memory_hard_limit=float(g[p + "memory_hard_limit"]))


def profile(lists, sc):
    """per list entry: (score, pad) -- what the reference fixes; ties may come in any order."""
    m = lists.shape[0]
    dense = sc.toarray()
    return np.where(lists >= 0, dense[np.arange(m)[:, None], np.maximum(lists, 0)], np.nan), lists < 0


@pytest.mark.parametrize("case", cases())
def test_oracle_reproduces_the_reference_lists(g, case):
    a = case_args(g, case)
    lists, modes, _, sc = so.recommend(**a)
    ref = g[case + "_recs"]
    s_mine, pad_mine = profile(lists, sc)
    s_ref, pad_ref = profile(ref, sc)
    np.testing.assert_array_equal(pad_mine, pad_ref)
    if case == "float":
        np.testing.assert_allclose(s_mine, s_ref, rtol=1e-12, atol=0)
    else:
        np.testing.assert_array_equal(s_mine, s_ref)
    np.testing.assert_array_equal(np.array(modes, dtype=np.int64), g[case + "_modes"])


def test_golden_covers_the_forms_the_model_meets(g):
    modes = np.concatenate([g[c + "_modes"] for c in cases()])
    assert set(modes[:, 2]) == {0, 1}                                      # dense and sparse chunks
    assert any((g[c + "_recs"] < 0).any() for c in cases())                # -1 padding
    rel = [relations(g, c) for c in cases()]
    assert any((r != r.T).nnz for r in rel) and any((r != r.T).nnz == 0 for r in rel)
    assert any(bool(g[c + "_implicit"]) for c in cases()) and any(bool(g[c + "_dense_output"]) for c in cases())


def test_dense_output_scores_with_s_on_csr_relations(g):
    """the recorded dense_output run ranks P S, not the P S^T of the sparse product, on non-symmetric relations."""
    a = case_args(g, "dense_output")
    assert (a["relations"] != a["relations"].T).nnz
    sc_s = so.recommend(**a)[3]
    sc_t = so.recommend(**dict(a, dense_output=False))[3]
    ref = g["dense_output_recs"]
    assert not np.array_equal(profile(ref, sc_s)[0], profile(ref, sc_t)[0])


def test_oracle_reproduces_the_wide_cooccurrence_run():
    w = np.load(WIDE)
    p = "wide_"
    lists, modes, _, sc = io.recommend(w[p + "train_idx"], w[p + "train_val"], tuple(w[p + "train_shape"]),
                                       w[p + "test_user"], w[p + "test_item"], w[p + "test_fdbk"],
                                       tuple(w[p + "test_shape"]), topk=int(w[p + "topk"]))
    np.testing.assert_array_equal(profile(lists, sc)[0], profile(w[p + "recs"], sc)[0])
    np.testing.assert_array_equal(np.array(modes, dtype=np.int64), w[p + "modes"])
    assert w[p + "train_shape"][1] > 30000


def test_sparse_matrix_refusal_takes_the_free_byte_count():
    from polara_b200.engine import cooc_csr_bytes, cooc_csr_memory_check
    n, nnz = 271_379, 123_456_789
    need = cooc_csr_bytes(nnz, n) + 1000
    assert cooc_csr_bytes(nnz, n) == 8 * (n + 1) + 12 * nnz
    assert cooc_csr_memory_check(nnz, n, 1000, need) == need
    with pytest.raises(MemoryError, match=r"271379 items with 123456789 stored entries takes %d bytes"
                       % cooc_csr_bytes(nnz, n)):
        cooc_csr_memory_check(nnz, n, 1000, need - 1)
    assert cooc_csr_memory_check(0, n, 0, 8 * (n + 1)) == 8 * (n + 1)

"""CPU checks of the item-to-item model against the reference's recorded runs (tests/golden/i2i_cases.npz, made by
oracle/make_i2i_golden.py): the f64 oracle's lists and chunk forms, the product-side chunk rule, the memory refusal of
the dense item x item matrix, and the metrics of padded lists."""
import os

import numpy as np
import pytest

from oracle import i2i_oracle as io

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "i2i_cases.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN, allow_pickle=False)


def cases():
    return [str(c) for c in np.load(GOLDEN)["cases"]]


def case_args(g, c):
    p = c + "_"
    return dict(train_idx=g[p + "train_idx"], train_val=g[p + "train_val"], train_shape=tuple(g[p + "train_shape"]),
                test_user=g[p + "test_user"], test_item=g[p + "test_item"], test_fdbk=g[p + "test_fdbk"],
                test_shape=tuple(g[p + "test_shape"]), topk=int(g[p + "topk"]), filter_seen=bool(g[p + "filter_seen"]),
                implicit=bool(g[p + "implicit"]), dense_output=bool(g[p + "dense_output"]),
                memory_hard_limit=float(g[p + "memory_hard_limit"]))


def row_profile(lists, sc, seen):
    """per list entry: (score, pad, seen) -- what the reference fixes; ties may come in any order."""
    m, k = lists.shape
    dense = sc.toarray()
    score = np.where(lists >= 0, dense[np.arange(m)[:, None], np.maximum(lists, 0)], np.nan)
    flag = np.zeros(lists.shape, dtype=bool)
    for u in range(m):
        flag[u] = np.isin(lists[u], seen.indices[seen.indptr[u]:seen.indptr[u + 1]]) & (lists[u] >= 0)
    return score, lists < 0, flag


def untied(score, sc):
    """positions whose score no other item of the row has (zero counts as a score of every unscored item)."""
    dense = sc.toarray()
    out = np.zeros(score.shape, dtype=bool)
    for u in range(score.shape[0]):
        vals, counts = np.unique(dense[u], return_counts=True)
        ok = np.isin(score[u], vals[counts == 1])
        out[u] = ok
    return out


def seen_csr(a):
    import scipy.sparse as sps
    return sps.csr_matrix((np.ones(len(a["test_user"])), (a["test_user"], a["test_item"])), shape=a["test_shape"][:2])


@pytest.mark.parametrize("case", cases())
def test_oracle_reproduces_the_reference_lists(g, case):
    a = case_args(g, case)
    lists, modes, nnz_u, sc = io.recommend(**a)
    ref = g[case + "_recs"]
    assert lists.shape == ref.shape
    s_mine, pad_mine, seen_mine = row_profile(lists, sc, seen_csr(a))
    s_ref, pad_ref, seen_ref = row_profile(ref, sc, seen_csr(a))
    np.testing.assert_array_equal(pad_mine, pad_ref)
    if case == "float":
        np.testing.assert_allclose(s_mine, s_ref, rtol=1e-12, atol=0)
    else:
        np.testing.assert_array_equal(s_mine, s_ref)
    # where no other item of the row has the same score, the reference fixes the item: same id, same seen flag
    fixed = untied(s_mine, sc) & ~pad_mine
    np.testing.assert_array_equal(seen_mine[fixed], seen_ref[fixed])
    np.testing.assert_array_equal(lists[fixed], ref[fixed])
    assert fixed.any()


@pytest.mark.parametrize("case", cases())
def test_oracle_chunk_forms_match_the_recorded_ones(g, case):
    a = case_args(g, case)
    _, modes, _, _ = io.recommend(**a)
    np.testing.assert_array_equal(np.array(modes, dtype=np.int64), g[case + "_modes"])


def test_golden_covers_both_forms_and_pads(g):
    modes = np.concatenate([g[c + "_modes"] for c in cases()])
    assert set(modes[:, 2]) == {0, 1}
    assert len(set(g["mixed_modes"][:, 2])) == 2 and len(g["mixed_modes"]) > 2
    assert (g["sparse_recs"] < 0).any()


@pytest.mark.parametrize("case", cases())
def test_product_chunk_rule_matches_the_oracle_on_the_golden_cases(g, case):
    from polara_b200.models import cooc_chunk_modes
    a = case_args(g, case)
    _, modes, nnz_u, _ = io.recommend(**a)
    got = cooc_chunk_modes(nnz_u, a["test_shape"][1], a["topk"], a["memory_hard_limit"], a["dense_output"])
    assert got == modes


@pytest.mark.parametrize("limit", [1, 0.25, 0.001, 0.00036])
def test_product_chunk_rule_at_the_threshold_edges(limit):
    """nnz equal to nnz_max or to half the block stays sparse; one more goes dense."""
    from polara_b200.models import cooc_chunk_modes, cooc_nnz_max
    assert cooc_nnz_max(1) == io.nnz_max(1)
    n_items, topk = 3000, 10
    for m in (1, 7, 1000, 50_000):
        try:
            a, b, _ = io.chunk_modes(np.zeros(m, np.int64), n_items, topk, limit)[0]
        except MemoryError:
            with pytest.raises(MemoryError):
                cooc_chunk_modes(np.zeros(m, np.int64), n_items, topk, limit)
            continue
        rows = b - a
        nnz_max = io.nnz_max(limit)
        for total in sorted({min(nnz_max, rows * n_items), nnz_max + 1, rows * n_items // 2, rows * n_items // 2 + 1,
                             0, rows * n_items}):
            nnz = np.zeros(m, np.int64)
            base, extra = divmod(total, rows)
            nnz[a:b] = base
            nnz[a:a + extra] += 1
            try:
                want = io.chunk_modes(nnz, n_items, topk, limit)
            except MemoryError:                   # no user chunk fits the limit (utils.py:44-47)
                with pytest.raises(MemoryError):
                    cooc_chunk_modes(nnz, n_items, topk, limit)
                break
            assert cooc_chunk_modes(nnz, n_items, topk, limit) == want
            assert want[0][2] == (total > nnz_max or total > 0.5 * rows * n_items)
            assert cooc_chunk_modes(nnz, n_items, topk, limit, dense_output=True) == [(x, y, True) for x, y, _ in want]


def test_dense_matrix_refusal_takes_the_free_byte_count():
    from polara_b200.engine import cooc_lds, cooc_memory_check
    n = 26744
    need = n * cooc_lds(n) * 8 + 1000
    assert cooc_memory_check(n, 1000, need) == need
    with pytest.raises(MemoryError, match=r"26744 items .* %d bytes" % (n * cooc_lds(n) * 8)):
        cooc_memory_check(n, 1000, need - 1)
    with pytest.raises(MemoryError):
        cooc_memory_check(200_000, 0, 80 << 30)


@pytest.mark.parametrize("case", cases())
def test_evaluate_lists_reproduces_the_reference_metrics(g, case):
    from polara_b200.host import evaluate_lists
    p = case + "_"
    names = [str(x) for x in g[p + "metric_names"]]
    lists = [(g[p + "recs"], g[p + "metrics"])]
    if p + "crafted_recs" in g:
        lists.append((g[p + "crafted_recs"], g[p + "crafted_metrics"]))
    for recs, want in lists:
        res = evaluate_lists(recs, g[p + "holdout_user"], g[p + "holdout_item"], g[p + "holdout_fdbk"],
                             int(g[p + "n_items_total"]), metric_type=["hits", "relevance", "ranking", "experience"])
        got = {"%s.%s" % (type(t).__name__, f): v for t in res for f, v in zip(t._fields, t) if v is not None}
        for name, value in zip(names, want):
            if name.startswith("Relevance.") or name == "Ranking.ndcg":
                continue    # averages over safe_divide, which leaves masked entries uninitialised (evaluation.py:18-20)
            assert got[name] == pytest.approx(value, rel=1e-12, abs=1e-15), (case, name)


def test_padded_lists_never_match_a_holdout_item():
    """a -1 pad of user 1 is no hit for the last item of user 0 (build_rank_matrix drops negative entries)."""
    from polara_b200.host import evaluate_lists
    hits = evaluate_lists(np.array([[0, 1], [-1, -1]]), np.array([0, 1]), np.array([4, 2]), None, 5, metric_type="hits")
    assert hits.true_positive == 0

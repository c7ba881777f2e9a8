"""The host restatement of the reference's unseen-item sampler (oracle/sampler_oracle.py) against the reference's own
draws recorded in tests/golden/sampler_cases.npz (oracle/make_sampler_golden.py): bit for bit on every case."""
import os

import numpy as np
import pytest
import scipy.sparse as sps

from oracle import sampler_oracle as so

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sampler_cases.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def _case(g, j):
    return (int(g["c%d_n" % j]), int(g["c%d_s" % j]), g["c%d_indptr" % j], g["c%d_indices" % j], g["c%d_seeds" % j],
            g["c%d_out" % j])


def test_fixture_covers_the_adversarial_shapes(g):
    n_cases = int(g["n_cases"])
    assert n_cases >= 9
    shapes = set()
    for j in range(n_cases):
        n, s, indptr, indices, seeds, _ = _case(g, j)
        shapes.add(n)
        lens = np.diff(indptr)
        if j != 1:
            assert (lens == 0).any()
            assert (n - lens == s).any()                    # a row with exactly s items left
        for u in range(len(lens)):
            row = indices[indptr[u]:indptr[u + 1]]
            if len(row) > 1 and (np.diff(row) < 0).any() and (np.diff(row) > 0).any():
                shapes.add("unsorted")
            if len(row) and (row >= n - len(row)).any():
                shapes.add("tail")
        assert seeds.dtype == np.uint32
    assert {255, 256, 257, 1023, 1024, 1025, "unsorted", "tail"} <= shapes
    assert int(g["c1_s"]) == 1
    assert {0, 2 ** 32 - 1} <= set(int(x) for x in g["c0_seeds"])


def test_restatement_equals_every_reference_case(g):
    for j in range(int(g["n_cases"])):
        n, s, indptr, indices, seeds, out = _case(g, j)
        got = so.sample_rows(indptr, indices, n, s, seeds)
        np.testing.assert_array_equal(got, out.astype(np.int64), err_msg="case %d" % j)


def test_mf_random_item_scoring_draws_the_same_items(g):
    n, s, indptr, indices, seeds, _ = _case(g, 0)
    items = so.sample_rows(indptr, indices, n, s, seeds)
    uf, vf = g["mf_user_factors"], g["mf_item_factors"]
    want = np.zeros(items.shape)
    for k in range(uf.shape[1]):                        # the reference's summation order
        want += uf[:, None, k] * vf[items, k]
    np.testing.assert_allclose(g["mf_scores"], want, rtol=1e-13, atol=1e-13)


def test_model_run_lists_and_draw(g):
    shape = tuple(int(x) for x in g["run_shape"])
    tu, ti, tf = g["run_test_user"], g["run_test_item"], g["run_test_fdbk"]
    keep = tf != 0
    profile = sps.csr_matrix((tf[keep], (tu[keep], ti[keep])), shape=shape)
    indptr, indices = so.exclusion_lists(profile, g["run_holdout_user"], g["run_holdout_item"], shape)
    np.testing.assert_array_equal(indptr, g["run_excl_indptr"])
    np.testing.assert_array_equal(indices, g["run_excl_indices"])
    seeds = np.random.SeedSequence(int(g["run_data_seed"])).generate_state(shape[0])
    np.testing.assert_array_equal(seeds, g["run_seeds"])
    got = so.sample_rows(indptr, indices, shape[1], int(g["run_n_unseen"]), seeds)
    np.testing.assert_array_equal(got, g["run_sampled"])
    e = profile.dot(g["run_item_factors"])
    np.testing.assert_allclose(so.sampled_scores(e, g["run_item_factors"], got), g["run_unseen_scores"], rtol=1e-10,
                               atol=1e-12)


def test_scipy_general_path_order_is_kept():
    profile = sps.csr_matrix((np.ones(3), [1, 5, 9], [0, 3]), shape=(1, 12))
    indptr, indices = so.exclusion_lists(profile, np.array([0, 0]), np.array([7, 3]), (1, 12))
    assert list(indices) == [3, 7, 9, 5, 1]


class _Words:
    def __init__(self, words):
        self.words = list(words)

    def next(self):
        return self.words.pop(0)


@pytest.mark.parametrize("j", [1, 2, 3, 5, 8, 13, 16, 20, 31])
def test_randrange_is_the_raw_stream_rule(j):
    for n in (2 ** j - 1, 2 ** j, 2 ** j + 1):
        if n <= 0:
            continue
        b = n.bit_length()
        stream = so.RawStream(12345 + n)
        ref = so.RawStream(12345 + n)
        for _ in range(200):
            r = so.randrange(stream, n)
            while True:
                w = ref.next() >> (32 - b)
                if w < n:
                    break
            assert r == w and 0 <= r < n
    # rejection: a word whose top b bits are >= n is skipped
    n = 5                                                 # b = 3: 5, 6, 7 are rejected
    assert so.randrange(_Words([7 << 29, 5 << 29, 4 << 29]), n) == 4
    with pytest.raises(ValueError, match="empty range"):
        so.randrange(so.RawStream(0), 0)


def test_raw_stream_is_init_genrand():
    # first output of MT19937 after init_genrand(5489), the generator's published default seed
    assert so.RawStream(5489).next() == 3499211612

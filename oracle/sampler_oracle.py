"""Host restatement of the reference's on-the-fly sampler of unseen items (polara/lib/sampler.py) -- TEST INFRASTRUCTURE.

Written from the semantics, not from the reference's code:

* numba's ``random.seed(s)`` is MT19937 ``init_genrand(s)``; its raw 32-bit stream after that is the raw stream of
  ``np.random.RandomState(s)`` (``randint(0, 2**32, dtype=np.uint32)`` returns it word for word).
* numba's ``random.randrange(n)`` (CPython flavour): ``b = n.bit_length()``; draw a word ``w``, take ``w >> (32 - b)``;
  draw again while that is ``>= n``.  ``n <= 0`` raises ``ValueError("empty range for randrange()")``.
* ``prime_sampler_state`` moves the excluded items to the tail of ``range(n)`` with two dicts (``state``: position ->
  item for the positions whose item moved, ``track``: item -> position for the items that moved), in LIST order;
  ``sample_fill`` then draws with ``randrange(remaining)`` and swaps the drawn position with the last live one.

Plain Python dicts reproduce those dict operations one for one.
"""
import numpy as np


class RawStream:
    """The MT19937 raw 32-bit stream after ``init_genrand(seed)``, read word by word."""

    CHUNK = 1024

    def __init__(self, seed):
        self._rs = np.random.RandomState(int(seed) & 0xFFFFFFFF)
        self._buf = np.empty(0, dtype=np.uint32)
        self._pos = 0

    def next(self):
        if self._pos == len(self._buf):
            self._buf = self._rs.randint(0, 2 ** 32, size=self.CHUNK, dtype=np.uint32)
            self._pos = 0
        w = int(self._buf[self._pos])
        self._pos += 1
        return w


def randrange(stream, n):
    n = int(n)
    if n <= 0:
        raise ValueError("empty range for randrange()")
    shift = 32 - n.bit_length()
    while True:
        r = stream.next() >> shift
        if r < n:
            return r


def prime(n, exclude):
    """position map after the excluded items (in list order) were moved to the tail of range(n)."""
    state, track = {}, {}
    last = n - 1
    for i, item in enumerate(exclude):
        item = int(item)
        pos = last - i
        x = track.get(item, item)       # where the item sits now
        t = state.get(pos, pos)         # what sits at the tail slot
        state[x] = t
        track[t] = x
        state.pop(pos, None)
        track.pop(item, None)
    return state


def sample_user(n, exclude, n_samples, seed):
    """the ``n_samples`` item ids the reference draws for one user (sample_row_wise / mf_random_item_scoring)."""
    state = prime(n, exclude)
    remaining = n - len(exclude)
    stream = RawStream(seed)
    out = np.empty(n_samples, dtype=np.int64)
    for k in range(n_samples):
        i = randrange(stream, remaining)
        out[k] = state.get(i, i)
        remaining -= 1
        state[i] = state.get(remaining, remaining)
        state.pop(remaining, None)
    return out


def sample_rows(indptr, indices, n, n_samples, seeds, rows=None):
    """``sample_row_wise`` for the given rows (all by default): int64 [len(rows) x n_samples]."""
    rows = range(len(indptr) - 1) if rows is None else rows
    return np.stack([sample_user(n, indices[indptr[u]:indptr[u + 1]], n_samples, seeds[u]) for u in rows]) \
        if len(rows) else np.empty((0, n_samples), dtype=np.int64)


def exclusion_lists(profile, holdout_user, holdout_item, shape):
    """``profile_matrix + matrix_from_observations(holdout)`` as RandomSampleEvaluationSVDMixin forms it (models.py:
    1145-1148, evaluation.py:45-61): a boolean holdout CSR whose rows are the runs of ``holdout_user`` and whose indices
    keep the holdout order, added to the profile CSR by scipy -- the result's index order is scipy's."""
    import scipy.sparse as sps
    keys = np.asarray(holdout_user)
    n_obs = len(keys)
    hm = sps.csr_matrix(shape, dtype=bool)
    hm.data = np.ones(n_obs, dtype=bool)
    hm.indices = np.asarray(holdout_item)
    hm.indptr = np.r_[0, np.where(np.diff(keys))[0] + 1, n_obs]
    s = profile + hm
    return s.indptr.astype(np.int64), s.indices.astype(np.int64)


def sampled_scores(user_factors, item_factors, items):
    """f64 scores of the sampled items (mf_random_item_scoring's inner loop)."""
    u = np.asarray(user_factors, dtype=np.float64)
    v = np.asarray(item_factors, dtype=np.float64)
    return np.einsum("ur,usr->us", u, v[items])

"""Host emulation of the item-to-item summation contract (DESIGN.md §3.5, §4 "Item-to-item model"), shared by the exact
item-to-item tests.

build_s         S = AᵀA as a dense fp64 array: every entry summed over the users in ascending order, one rounded add
                per user (the product of two fp32 values is exact in fp64), then a zero diagonal;
scores          s_u = Σ_i p_ui·M[i, :] over the stored entries of M, i ascending: a rounded product, then a rounded add.
                M is S for the item-to-item model, Sᵀ or S for SimilarityAggregation (oracle/sim_oracle.scoring_operand);
expected_lists  nnz_u, the dense-rule and the sparse-rule lists (oracle/i2i_oracle) and the dense lists' scores;
cooc_fixture, sim_fixture, scoring_users
                training data, relations and test users whose sums depend on the order, with extras at the kernels'
                boundaries (see their docstrings);
cooc_case, wide_case, sim_case
                the fixed-seed cases the tests share, with their emulated S and scores.

``order="desc"`` runs either sum in the reverse order.  It serves only to show that a fixture tells the orders apart:
on integer data every order gives the same bits."""
import functools

import numpy as np
import scipy.sparse as sps

from oracle import i2i_oracle as io
from oracle import sim_oracle as so

HASH_WORK = 512        # csrc/i2i.cu kHashWork: rows / users with more work take the global-row path
BUILD_BATCH = 128      # csrc/i2i.cu kBuildBatch: users staged per batch by the build kernels
SCORE_BATCH = 32       # test items a scoring warp loads per batch (pb200_i2i_topk)
SCORE_PANEL = 256      # columns of one sweep panel of pb200_i2i_topk (32 * kScoreR)


def fp32_values(rng, size, lo=-20, hi=20):
    """fp32-representable values: random 24-bit mantissas, exponents lo..hi, both signs."""
    mant = rng.integers(1 << 23, 1 << 24, size).astype(np.float64)
    return rng.choice([-1.0, 1.0], size) * np.ldexp(mant, rng.integers(lo, hi + 1, size) - 23)


def _csr(x):
    x = sps.csr_matrix(x, dtype=np.float64, copy=True)
    x.sum_duplicates()
    x.sort_indices()
    return x


def build_s(a, implicit=False, order="asc", rows=None):
    """rows ``rows`` (default all) of S = AᵀA with a zero diagonal, dense fp64 ``[len(rows) x n]``: for the users in
    ``order``, S[i, j] = S[i, j] + a_ui·a_uj."""
    a = _csr(a)
    m, n = a.shape
    rows = np.arange(n) if rows is None else np.asarray(rows, np.int64)
    pos = np.full(n, -1, np.int64)
    pos[rows] = np.arange(len(rows))
    out = np.zeros((len(rows), n))
    for u in (range(m) if order == "asc" else range(m - 1, -1, -1)):
        c, v = a.indices[a.indptr[u]:a.indptr[u + 1]], a.data[a.indptr[u]:a.indptr[u + 1]]
        if implicit:
            v = np.sign(v)
        r = pos[c] >= 0
        if r.any():
            out[np.ix_(pos[c[r]], c)] += np.outer(v[r], v)      # distinct items: one rounded add per entry
    out[np.arange(len(rows)), rows] = 0.0
    return out


def csr_of(dense):
    """the CSR of a dense S without its zeros (setdiag(0) is already applied), indices ascending."""
    c = sps.csr_matrix(dense)
    c.eliminate_zeros()
    c.sort_indices()
    return c


def scores(p, mat, order="asc"):
    """dense fp64 ``[m x n]`` scores P·M: per user acc = acc + p_ui·M[i, :] over the stored entries of row i of M, the
    items i in ``order``."""
    p, mat = _csr(p), _csr(mat)
    out = np.zeros((p.shape[0], mat.shape[1]))
    for u in range(p.shape[0]):
        q = range(p.indptr[u], p.indptr[u + 1])
        acc = out[u]
        for t in (q if order == "asc" else reversed(q)):
            i, x = p.indices[t], p.data[t]
            lo, hi = mat.indptr[i], mat.indptr[i + 1]
            c = mat.indices[lo:hi]
            acc[c] = acc[c] + x * mat.data[lo:hi]
    return out


def expected_lists(sc, seen, k, filter_seen):
    """``(nnz int64 [m], dense int64 [m x k], sparse int64 [m x k], dense scores f64 [m x k])`` of the dense score block
    ``sc`` under the oracle's rules; ``seen`` is the CSR of every test triplet."""
    m = sc.shape[0]
    dense, sparse = np.empty((m, k), np.int64), np.empty((m, k), np.int64)
    for u in range(m):
        row = sc[u]
        dense[u] = io.dense_rule(row, seen.indices[seen.indptr[u]:seen.indptr[u + 1]], k, filter_seen)
        nz = np.flatnonzero(row)
        sparse[u] = io.sparse_rule(nz, row[nz], k)
    return (sc != 0).sum(axis=1).astype(np.int64), dense, sparse, np.take_along_axis(sc, dense, axis=1)


def build_work(a):
    """work of each item row: Σ over its users of their row lengths (csrc/i2i.cu row_work_kernel)"""
    a = _csr(a)
    a.data[:] = 1.0
    return np.asarray(a.T @ np.diff(a.indptr).astype(np.float64)).astype(np.int64)


def score_work(p, mat):
    """work of each test user: Σ over its items of the stored entries of their rows of M"""
    p, mat = _csr(p), _csr(mat)
    p.data[:] = 1.0
    return np.asarray(p @ np.diff(mat.indptr).astype(np.float64)).astype(np.int64)


def differs(x, y):
    """entries whose bits differ"""
    return np.asarray(x).view(np.int64) != np.asarray(y).view(np.int64)


# ---- fixtures ----------------------------------------------------------------------------------------------------------
def _strata(rng, free, count):
    """``count`` ids of the sorted array ``free``, one from each of ``count`` equal slices: spread over every panel"""
    edges = np.linspace(0, len(free), count + 1).astype(np.int64)
    return np.array([free[rng.integers(edges[t], edges[t + 1])] for t in range(count)])


def cooc_fixture(n_items, seed, n_base=400, n_pool=60, n_mid=100):
    """Training data for S = AᵀA.  Returns ``(a, roles)``: ``a`` a user x item CSR of fp32-representable values.

    * base users rate each of ``n_pool`` pool items with probability 0.4 (so a pool pair has about 60 co-raters), 2 to 8
      tail items, and the mid items: each mid item has 6 to 12 raters, so its row sums 3 or more terms against most
      pool items at a work of about 200-400, on the table path;
    * three heavy users rate 150, 200 and 300 items: more than one item per thread of a 128-thread build CTA;
    * ``cancel``: pairs (i, j) rated only by two users, with values (a, b) and (a, -b): S[i, j] is exactly 0;
    * ``dup``: pairs (x, y) of identical columns (5 raters), with low ids: S[x, :] = S[y, :] off x and y;
    * ``raters``: items with exactly 128, 129 and 257 raters (the build's staging batch);
    * ``work``: items whose work is exactly 512 and 513 (16 users of 32 items, 19 users of 27 items);
    * the last 5 % of the tail is never rated."""
    rng = np.random.default_rng(seed)
    ids = rng.permutation(np.arange(n_items // 10))
    dup = ids[:4].reshape(2, 2)
    dup.sort(axis=1)
    free = np.setdiff1d(np.arange(n_items), dup.ravel())
    pool = _strata(rng, free, n_pool)
    free = rng.permutation(np.setdiff1d(free, pool))
    cancel = np.sort(free[:6].reshape(3, 2), axis=1)
    raters = dict(zip((128, 129, 257), free[6:9]))
    work = dict(zip((512, 513), free[9:11]))
    mid = np.sort(free[11:11 + n_mid])
    tail = np.sort(free[11 + n_mid:])
    tail = tail[:len(tail) - len(tail) // 20]
    u, i = [], []

    def rate(user, items):
        u.extend([user] * len(items))
        i.extend(items)
    for b in range(n_base):
        rate(b, pool[rng.random(n_pool) < 0.4])
        rate(b, rng.choice(tail, rng.integers(2, 9), replace=False))
    for it in mid:
        for b in rng.choice(n_base, rng.integers(6, 13), replace=False):
            rate(b, [it])
    for c, r in raters.items():
        for b in rng.choice(n_base, c, replace=False):
            rate(b, [r])
    for x, _ in dup:
        for b in rng.choice(n_base, 5, replace=False):
            rate(b, [x])
    user = n_base
    heavy = []
    for deg in (150, 200, 300):
        rate(user, np.r_[pool, rng.choice(tail, deg - n_pool, replace=False)])
        heavy.append(user)
        user += 1
    for target, (n_u, deg) in ((512, (16, 32)), (513, (19, 27))):
        for _ in range(n_u):
            rate(user, np.r_[work[target], rng.choice(pool, deg - 1, replace=False)])
            user += 1
    vals = fp32_values(rng, len(u))
    u, i = np.asarray(u), np.asarray(i)
    for x, y in dup:                                   # y: a copy of column x
        sel = i == x
        u, i, vals = np.r_[u, u[sel]], np.r_[i, np.full(sel.sum(), y)], np.r_[vals, vals[sel]]
    for ci, cj in cancel:
        b1, b2 = rng.choice(n_base, 2, replace=False)
        a_, b_ = fp32_values(rng, 2)
        u, i, vals = np.r_[u, b1, b1, b2, b2], np.r_[i, ci, cj, ci, cj], np.r_[vals, a_, b_, a_, -b_]
    a = sps.csr_matrix((vals, (u, i)), shape=(user, n_items))
    assert a.nnz == len(vals)                          # no (user, item) pair twice
    roles = dict(pool=pool, mid=mid, tail=tail, dup=dup, cancel=cancel, raters=raters, work=work, heavy=heavy)
    return _csr(a), roles


def _exact_work_items(rng, nnz, items, target, min_items=3):
    """``min_items`` or more distinct ``items`` whose row counts ``nnz`` sum to exactly ``target``"""
    by = {}
    for it in items:
        by.setdefault(int(nnz[it]), []).append(int(it))
    for _ in range(20000):
        pick, tot = [], 0
        for it in rng.permutation(items):
            rest = [x for x in by.get(target - tot, ()) if x not in pick]
            if len(pick) >= min_items - 1 and rest:
                return sorted(pick + [rest[0]])
            if tot + nnz[it] < target and nnz[it] > 0:
                pick.append(int(it))
                tot += int(nnz[it])
    raise AssertionError("no item set of work %d" % target)


def scoring_users(mat, heavy_items, light_items, seed, n_heavy=40, n_light=150, dup=()):
    """Test triplets ``(user, item, fdbk)`` scored against the rows of ``mat`` (the scoring operand), their shape and
    their roles.

    Users 0..n_heavy-1 take 3 to 8 ``heavy_items`` (rows of many entries) and up to 30 others; four of them 40 to 70
    items (more than one scoring batch of 32): the global-row path.  Then the cancellation users, three per ``dup``
    pair (x, y): +q on x and -q on y, so that every score outside row x cancels to exactly 0, and nothing more, or one
    or three ``light_items`` after y: exact zeros among nonzero scores.  Then ``n_light`` users of 4 to 7
    ``light_items`` with work at most 512 (the table path), two users of work exactly 512 and 513, one with only zero
    feedback and one with nothing.  About 3 % of the light triplets have zero feedback: seen, not in P."""
    rng = np.random.default_rng(seed)
    mat = _csr(mat)
    nnz = np.diff(mat.indptr)
    n_items = mat.shape[1]
    others = np.setdiff1d(np.arange(n_items), heavy_items)
    rows, roles = [], dict(heavy=[], cancel=[], light=[], work={})

    def add(items, vals, role):
        rows.append((np.asarray(items, np.int64), np.asarray(vals, np.float64)))
        roles[role].append(len(rows) - 1)
    for h in range(n_heavy):
        extra = rng.integers(40, 71) if h % 10 == 3 else rng.integers(0, 31)
        items = np.r_[rng.choice(heavy_items, rng.integers(3, 9), replace=False), rng.choice(others, extra, replace=False)]
        add(items, fp32_values(rng, len(items), -10, 10), "heavy")
    for x, y in dup:
        later = rng.permutation(light_items[light_items > y])
        for n_after in (0, 1, 3):
            q = fp32_values(rng, 1, -10, 10)[0]
            add(np.r_[x, y, later[:n_after]], np.r_[q, -q, fp32_values(rng, n_after, -10, 10)], "cancel")
    for _ in range(n_light):
        items = rng.choice(light_items, rng.integers(4, 8), replace=False)
        while nnz[items].sum() > HASH_WORK:
            items = items[:-1]
        add(items, fp32_values(rng, len(items), -10, 10), "light")
    for target in (HASH_WORK, HASH_WORK + 1):
        items = _exact_work_items(rng, nnz, light_items, target)
        rows.append((np.asarray(items, np.int64), fp32_values(rng, len(items), -10, 10)))
        roles["work"][target] = len(rows) - 1
    rows.append((rng.choice(light_items, 2, replace=False), np.zeros(2)))
    rows.append((np.zeros(0, np.int64), np.zeros(0)))
    user = np.concatenate([np.full(len(it), u) for u, (it, _) in enumerate(rows)])
    item = np.concatenate([it for it, _ in rows]).astype(np.int64)
    fdbk = np.concatenate([f for _, f in rows])
    light = np.isin(user, roles["light"])
    fdbk[light & (rng.random(len(fdbk)) < 0.03)] = 0.0
    return (user, item, fdbk), (len(rows), n_items), roles


def scoring_matrices(triplets, shape):
    """``(P, seen)``: P as the item-to-item model reads it (zero feedback dropped) and the CSR of every triplet."""
    user, item, fdbk = triplets
    seen = sps.csr_matrix((np.ones(len(user)), (user, item)), shape=shape)
    return _csr(io.test_matrix(user, item, fdbk, shape)), seen


def sim_fixture(n_items, seed, n_pool=60):
    """Non-symmetric item relations with arbitrary fp64 values (not fp32-representable; exponents 2⁻²⁰..2²⁰, both
    signs) and a unit diagonal: the rows and columns of ``n_pool`` pool items are half full, and 1 % of the rest.
    Returns ``(relations CSR, pool)``."""
    rng = np.random.default_rng(seed)
    pool = _strata(rng, np.arange(n_items), n_pool)
    dense = np.zeros((n_items, n_items), bool)
    dense[pool] = rng.random((n_pool, n_items)) < 0.5
    dense[:, pool] |= rng.random((n_items, n_pool)) < 0.5
    dense |= rng.random((n_items, n_items)) < 0.01
    r, c = np.nonzero(dense)
    vals = rng.standard_normal(len(r)) * np.exp2(rng.integers(-20, 21, len(r)))
    rel = sps.csr_matrix((np.r_[vals, np.ones(n_items)], (np.r_[r, np.arange(n_items)], np.r_[c, np.arange(n_items)])),
                         shape=(n_items, n_items))
    return _csr(rel), pool


# ---- the shared cases ----------------------------------------------------------------------------------------------------
COOC_ITEMS = 1500          # five full 256-column sweep panels and a partial one
WIDE_ITEMS = 8192 + 333    # two build panels at the full width of 8192 columns, the last one partial
SIM_ITEMS = 1200


@functools.lru_cache(maxsize=None)
def cooc_case():
    """the item-to-item case: training data, S (dense and CSR), the test users, P, seen and the emulated scores"""
    a, roles = cooc_fixture(COOC_ITEMS, 1)
    s = build_s(a)
    s_csr = csr_of(s)
    triplets, shape, users = scoring_users(s_csr, roles["pool"], roles["mid"], 2, dup=roles["dup"])
    p, seen = scoring_matrices(triplets, shape)
    return dict(a=a, roles=roles, s=s, s_csr=s_csr, triplets=triplets, shape=shape, users=users, p=p, seen=seen,
                scores=scores(p, s_csr))


@functools.lru_cache(maxsize=None)
def wide_case():
    """training data of WIDE_ITEMS items and the emulated rows of S at the pool items, the boundary items and 100
    others"""
    a, roles = cooc_fixture(WIDE_ITEMS, 5)
    rng = np.random.default_rng(6)
    rows = np.unique(np.r_[roles["pool"], list(roles["raters"].values()), list(roles["work"].values()),
                           roles["cancel"].ravel(), roles["dup"].ravel(), rng.choice(WIDE_ITEMS, 100, replace=False)])
    return dict(a=a, roles=roles, rows=rows, s=build_s(a, rows=rows))


@functools.lru_cache(maxsize=None)
def sim_case(dense_output):
    """SimilarityAggregation: the relations, the scoring operand M (Sᵀ, or S with ``dense_output``), the test users,
    P, seen and the emulated scores"""
    rel, pool = sim_fixture(SIM_ITEMS, 3)
    mat = _csr(so.scoring_operand(so.similarity_matrix(rel), dense_output))
    triplets, shape, users = scoring_users(mat, pool, np.setdiff1d(np.arange(SIM_ITEMS), pool), 4)
    p, seen = scoring_matrices(triplets, shape)
    return dict(rel=rel, pool=pool, mat=mat, triplets=triplets, shape=shape, users=users, p=p, seen=seen,
                scores=scores(p, mat))


MODEL_LIMIT = 0.0003       # memory_hard_limit of the model case: nine chunks of 22 or 23 test users


@functools.lru_cache(maxsize=None)
def model_case():
    """the item-to-item model on the training data of cooc_case: its 40 heavy test users (score blocks more than half
    full: dense chunks), then 160 users of one or two tail items (few nonzero scores: sparse chunks)"""
    c = cooc_case()
    rng = np.random.default_rng(7)
    user, item, fdbk = c["triplets"]
    keep = np.isin(user, c["users"]["heavy"])
    user, item, fdbk = [user[keep]], [item[keep]], [fdbk[keep]]
    n_heavy = len(c["users"]["heavy"])
    for u in range(n_heavy, n_heavy + 160):
        items = rng.choice(c["roles"]["tail"], rng.integers(1, 3), replace=False)
        user.append(np.full(len(items), u))
        item.append(items)
        fdbk.append(fp32_values(rng, len(items), -10, 10))
    triplets = np.concatenate(user), np.concatenate(item), np.concatenate(fdbk)
    shape = (n_heavy + 160, COOC_ITEMS)
    p, seen = scoring_matrices(triplets, shape)
    return dict(triplets=triplets, shape=shape, p=p, seen=seen, scores=scores(p, c["s_csr"]))

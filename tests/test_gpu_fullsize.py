"""Parity at the full C2 size (1 M users x 100 K items, 1e8 interactions, rank 50, top-10) through
size-independent properties -- the oracle cannot score 1e11 pairs, so the whole result is checked by invariants and a
random sample of user rows is checked against f64 scores computed on the host:

  * every list: ids in range and distinct, scores non-increasing, NO seen item anywhere (checked for all 1e7 entries);
  * sampled rows: a valid top-k of the f64 scores (order contract of models.py:494-519 + 561-563), reported scores
    equal the canonical scores of the reported items;
  * the exact fp32 SIMT kernel and the tensor-core kernel agree bit for bit on all 1 M rows;
  * item-sharded scoring + k-way merge equals the unsharded result (all rows);
  * a second run is bit-identical (fixed summation and insertion order).
"""
import os
import sys

import numpy as np
import pytest
import torch

from tests.helpers import check_topk_against_scores

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

M, N, NNZ, R, K = 1_000_000, 100_000, 100_000_000, 50, 10


@pytest.fixture(scope="module")
def c2():
    from polara_b200.engine import DeviceCSR, get_engine
    sys.path.insert(0, ROOT)
    from bench import synth_csr_torch
    if torch.cuda.get_device_properties(0).total_memory < 60e9:
        pytest.skip("needs a large-memory GPU")
    eng = get_engine(0)
    dev = eng.device
    indptr, indices, values = synth_csr_torch(M, N, NNZ, 20260924, dev)
    # item factors with a popularity-like norm profile (what a trained SVD gives), fixed seed
    g = torch.Generator(device=dev); g.manual_seed(7)
    scale = (1.0 / torch.arange(1, N + 1, device=dev, dtype=torch.float32)) ** 0.35
    scale = scale[torch.randperm(N, generator=g, device=dev)]
    v = torch.zeros((N, 64), device=dev)
    v[:, :R] = torch.randn((N, R), generator=g, device=dev) * scale[:, None] * (0.93 ** torch.arange(R, device=dev))
    p = DeviceCSR(indptr, indices, values, (M, N))
    e = eng.spmm(p, v, ell=R)
    eng.set_score_kernel("tc")
    ids, sc = eng.score_topk(e, v, R, K, seen=(indptr, indices), want_scores=True)
    torch.cuda.synchronize()
    yield dict(eng=eng, p=p, v=v, e=e, ids=ids, sc=sc)
    eng.set_score_kernel("tc")


def test_fullsize_list_invariants(c2):
    ids, sc, p = c2["ids"], c2["sc"], c2["p"]
    assert ids.shape == (M, K) and int(ids.min()) >= 0 and int(ids.max()) < N
    srt = torch.sort(ids, dim=1).values
    assert bool((srt[:, 1:] != srt[:, :-1]).all()), "duplicate item inside a list"
    assert bool((sc[:, 1:] <= sc[:, :-1]).all()), "scores must be non-increasing along a list"
    assert bool(torch.isfinite(sc).all())
    # no seen item in any list: (user, item) keys of the lists against the sorted keys of the interactions
    rows = torch.repeat_interleave(torch.arange(M, device=ids.device), p.indptr[1:] - p.indptr[:-1])
    seen_keys = rows * N + p.indices.to(torch.int64)                # sorted: CSR rows ascending, columns ascending
    del rows
    rec_keys = (torch.arange(M, device=ids.device)[:, None] * N + ids).reshape(-1)
    pos = torch.searchsorted(seen_keys, rec_keys).clamp_(max=seen_keys.numel() - 1)
    assert not bool((seen_keys[pos] == rec_keys).any()), "a seen item was recommended"


def test_fullsize_sampled_rows_against_f64(c2):
    eng, p, v, e, ids, sc = (c2[k] for k in ("eng", "p", "v", "e", "ids", "sc"))
    rng = np.random.default_rng(3)
    users = np.sort(rng.choice(M, size=192, replace=False))
    ut = torch.from_numpy(users).to(e.device)
    e_h = e[ut][:, :R].cpu().numpy().astype(np.float64)
    v_h = v[:, :R].cpu().numpy().astype(np.float64)
    s64 = e_h @ v_h.T
    ip = p.indptr.cpu().numpy()
    ix = p.indices.cpu().numpy()
    rows = np.concatenate([np.full(ip[u + 1] - ip[u], i) for i, u in enumerate(users)])
    cols = np.concatenate([ix[ip[u]:ip[u + 1]] for u in users])
    tol = 4e-6 * np.abs(e_h).sum(1).max() * np.abs(v_h).max()
    frac = check_topk_against_scores(ids[ut].cpu().numpy(), s64, rows, cols, K, tol)
    assert frac > 0.99
    got = np.take_along_axis(s64, ids[ut].cpu().numpy(), axis=1)
    np.testing.assert_allclose(sc[ut].cpu().numpy(), got, atol=tol)


def test_fullsize_kernels_agree_and_rerun_is_identical(c2):
    eng, p, v, e, ids, sc = (c2[k] for k in ("eng", "p", "v", "e", "ids", "sc"))
    again, sc_again = eng.score_topk(e, v, R, K, seen=(p.indptr, p.indices), want_scores=True)
    assert torch.equal(again, ids) and torch.equal(sc_again, sc)
    eng.set_score_kernel("simt")
    try:
        exact, sc_exact = eng.score_topk(e, v, R, K, seen=(p.indptr, p.indices), want_scores=True)
    finally:
        eng.set_score_kernel("tc")
    assert torch.equal(exact, ids), "tensor-core filter + rescoring differs from the exact fp32 kernel"
    assert torch.equal(sc_exact, sc)


def test_fullsize_sharded_merge_equals_unsharded(c2):
    eng, p, v, e, ids = (c2[k] for k in ("eng", "p", "v", "e", "ids"))
    bounds = [0, 33_333, 70_001, N]
    parts = [eng.score_topk_cands(e, v[lo:hi], R, K, seen=(p.indptr, p.indices), item_offset=lo)
             for lo, hi in zip(bounds[:-1], bounds[1:])]
    merged = eng.merge_cands(torch.stack(parts).contiguous(), len(parts), M, K)
    assert torch.equal(merged, ids)


def test_fullsize_build_properties(c2):
    """Truncated SVD of the full C2 matrix (what SVDModel.build computes, models.py:835-855): orthonormal item factors,
    descending positive singular values, small Ritz residuals ||A^T A v - sigma^2 v|| / sigma^2 for the leading
    triplets, and a second build is bit-identical."""
    eng, p = c2["eng"], c2["p"]
    at = eng.transpose(p)
    v, sigma, _, iters = eng.rsvd(p, at, R, 96, max_iters=12, tol=1e-7, seed=1)
    s = sigma.cpu().numpy()
    assert np.all(np.isfinite(s)) and np.all(s > 0) and np.all(np.diff(s) <= 0)
    vr = v[:, :R].double()
    gram = (vr.T @ vr).cpu().numpy()
    assert np.abs(gram - np.eye(R)).max() < 1e-4
    av = eng.spmm(p, v, ell=R)
    atav = eng.spmm(at, av, ell=R)[:, :R].double()
    s2 = torch.from_numpy(s ** 2).to(atav.device)
    resid = ((atav - vr * s2).norm(dim=0) / s2).cpu().numpy()
    assert resid[:5].max() < 5e-2, resid[:10]
    # |A v_j| = sigma_j
    np.testing.assert_allclose(av[:, :R].double().norm(dim=0).cpu().numpy(), s, rtol=1e-4)
    v2, sigma2, _, iters2 = eng.rsvd(p, at, R, 96, max_iters=12, tol=1e-7, seed=1)
    assert iters2 == iters and torch.equal(v2, v) and torch.equal(sigma2, sigma)


def test_fullsize_coffee_c4_properties():
    """C4 shape (1 M users x 50 K items x 5 feedback levels, ~5e7 interactions, core (60, 60, 4)): HOOI invariants
    (lib/tensor.py:37-96) and CoFFee scoring (models.py:1042-1054) against the oracle on sampled users."""
    from polara_b200.host import ArrayData
    from polara_b200.models import B200CoffeeModel
    sys.path.insert(0, ROOT)
    from bench import synth_csr_torch
    from oracle import polara_oracle as po
    if torch.cuda.get_device_properties(0).total_memory < 60e9:
        pytest.skip("needs a large-memory GPU")
    dev = torch.device("cuda", 0)
    U, I, F = 1_000_000, 50_000, 5
    indptr, indices, values = synth_csr_torch(U, I, 62_000_000, 7, dev)
    nnz = int(indices.shape[0])
    assert nnz > 45_000_000
    rows = torch.repeat_interleave(torch.arange(U, device=dev), indptr[1:] - indptr[:-1])
    idx = torch.stack([rows, indices.to(torch.int64), (values - 1).to(torch.int64)], 1).cpu().numpy()
    m_test = 100_000                                   # test users = the first 100 K users (known-user scenario)
    hi = int(indptr[m_test])
    del rows, values
    data = ArrayData(idx, np.ones(nnz), (U, I, F), idx[:hi, 0], idx[:hi, 1], idx[:hi, 2], (m_test, I, F), n_feedback=F)
    model = B200CoffeeModel(data)
    model.verbose = False
    model.mlrank, model.seed, model.num_iters = (60, 60, 4), 0, 4
    model.build()
    f = data.fields
    trace = np.asarray(model.core_norm_trace)
    assert len(trace) >= 2 and np.all(np.diff(trace) >= -1e-3 * trace[:-1]), trace     # ALS never loses captured norm
    core = model.factors["core"]
    assert core.shape == (60, 60, 4)
    np.testing.assert_allclose(np.linalg.norm(core), trace[-1], rtol=1e-3)
    assert np.linalg.norm(core) ** 2 <= nnz * (1 + 1e-4)                                # a projection of a 0/1 tensor
    for key in (f.userid, f.itemid, f.feedback):
        u = model.factors[key]
        assert np.abs(u.T @ u - np.eye(u.shape[1])).max() < 2e-3, key
    recs = model.get_recommendations()
    assert recs.shape == (m_test, 10) and recs.min() >= 0 and recs.max() < I
    srt = np.sort(recs, axis=1)
    assert (srt[:, 1:] != srt[:, :-1]).all()
    seen_keys = np.unique(idx[:hi, 0] * I + idx[:hi, 1])
    rec_keys = (np.arange(m_test)[:, None] * I + recs).ravel()
    assert not np.isin(rec_keys, seen_keys).any(), "a seen item was recommended"
    # sampled users against the oracle's scoring with the same factors
    rng = np.random.default_rng(1)
    users = np.sort(rng.choice(m_test, size=48, replace=False))
    ip = indptr.cpu().numpy()
    sel = np.concatenate([np.arange(ip[u], ip[u + 1]) for u in users])
    local = np.repeat(np.arange(len(users)), [ip[u + 1] - ip[u] for u in users])
    v, w = model.factors[f.itemid], model.factors[f.feedback]
    s64 = po.coffee_slice_scores(local, idx[sel, 1], idx[sel, 2], len(users), v, w, None)
    tol = 2e-5 * np.abs(s64).max()
    frac = check_topk_against_scores(recs[users], s64, local, idx[sel, 1], 10, tol)
    assert frac > 0.97

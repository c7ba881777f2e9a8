"""A numpy/scipy stand-in for a CHOLMOD factor (scikit-sparse ``sksparse.cholmod``)  --  TEST INFRASTRUCTURE.

The reference's HybridSVD (polara/recommender/hybrid/models.py) factorises ``S + beta I`` with
``sksparse.cholmod.cholesky(S, beta=beta)`` and reads the factor through polara's ``CholeskyFactor``
(polara/lib/cholesky.py): ``L()``, ``P()``, ``apply_P``, ``apply_Pt``, ``solve_Lt`` and ``cholesky_inplace``.  This module
provides exactly those, with CHOLMOD's conventions

    L L^T = P (S + beta I) P^T,   apply_P(v) = v[p],   apply_Pt = its inverse,

so that the real reference runs without scikit-sparse.  The factorisation is a dense Cholesky (test sizes only) of the
matrix permuted by reverse Cuthill-McKee (``scipy.sparse.csgraph``), a non-identity fill-reducing order, so that every
use of P is exercised.  L comes back sparse (CSC, as CHOLMOD returns it) with the exact zeros dropped.
"""
import numpy as np
import scipy.linalg
import scipy.sparse as sps
from scipy.sparse.csgraph import reverse_cuthill_mckee


class Factor:
    """``sksparse.cholmod.Factor`` restricted to what polara's CholeskyFactor calls."""

    def __init__(self, a, beta=0.0):
        self.cholesky_inplace(a, beta)

    def cholesky_inplace(self, a, beta=0.0):
        a = sps.csr_matrix(a, dtype=np.float64)
        n = a.shape[0]
        pattern = sps.csr_matrix(a + sps.eye(n, format="csr"))
        self._p = np.asarray(reverse_cuthill_mckee(pattern, symmetric_mode=True), dtype=np.int64)
        self._pinv = np.empty_like(self._p)
        self._pinv[self._p] = np.arange(n)
        dense = a.toarray() + beta * np.eye(n)
        low = np.linalg.cholesky(dense[np.ix_(self._p, self._p)])
        self._L = sps.csc_matrix(low)
        self._L.eliminate_zeros()

    def L(self):
        return self._L.copy()

    def P(self):
        return self._p.copy()

    def apply_P(self, b):
        """rows of b (dense or sparse, as CHOLMOD accepts both) in the order p."""
        return (sps.csr_matrix(b) if sps.issparse(b) else np.asarray(b))[self._p]

    def apply_Pt(self, b):
        return (sps.csr_matrix(b) if sps.issparse(b) else np.asarray(b))[self._pinv]

    def solve_Lt(self, b, use_LDLt_decomposition=True):
        if use_LDLt_decomposition:
            raise NotImplementedError("the stub holds an LL^T factor only")
        return scipy.linalg.solve_triangular(self._L.toarray().T, np.asarray(b, dtype=np.float64), lower=False)


def cholesky(a, beta=0.0):
    """``sksparse.cholmod.cholesky(A, beta)``: the factor of ``A + beta I``."""
    return Factor(a, beta)

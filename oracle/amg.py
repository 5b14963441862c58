"""TEST INFRASTRUCTURE ONLY. NumPy/SciPy restatement of the algebraic coarse solvers of palace_b200/csrc/b2p_amg.cu:
smoothed-aggregation AMG (strength, three-pass greedy aggregation, Jacobi-smoothed prolongation, Galerkin products, dense LDL^T
pseudo-inverse of the coarsest level, l1-Jacobi V-cycle) and AMS cycle type 14 with Pi built from G and the vertex coordinates.

The library keeps every sparse product in row-by-row (Gustavson) order with exact zeros dropped and sorted columns, which is
what scipy's CSR product does on operands with sorted columns; the scalar steps below use the same operations in the same
order. The aggregation therefore sees the same numbers and the hierarchies agree level by level, rows and entries."""
from __future__ import annotations

import math

import numpy as np
import scipy.linalg as sla
import scipy.sparse as sp

THETA = 0.08
COARSE_ROWS = 500
MAX_LEVELS = 10
MAX_KEEP = 0.8
PIVOT_TOL = 1e-12


def _sorted(A):
    A = sp.csr_matrix(A)
    A.sort_indices()
    return A


def _mul(A, B):
    return _sorted(A @ B)


def _transpose(A):
    return _sorted(A.T.tocsr())


def _abs_row_sums(A):
    return abs(A) @ np.ones(A.shape[1])  # sequential over the row's entries, as the library sums them


def aggregate(A):
    """Three-pass greedy aggregation in increasing row order; -1 for nodes without a strong neighbour."""
    n = A.shape[0]
    d = A.diagonal()
    rows = np.repeat(np.arange(n), np.diff(A.indptr))
    cols, vals = A.indices, A.data
    strong = (cols != rows) & (vals != 0.0) & (np.abs(vals) >= THETA * np.sqrt(np.abs(d[rows] * d[cols])))
    nbr = [cols[A.indptr[i]:A.indptr[i + 1]][strong[A.indptr[i]:A.indptr[i + 1]]] for i in range(n)]
    mag = [np.abs(vals[A.indptr[i]:A.indptr[i + 1]][strong[A.indptr[i]:A.indptr[i + 1]]]) for i in range(n)]
    agg = np.full(n, -1, dtype=np.int64)
    n_agg = 0
    for i in range(n):  # 1: roots with an untouched strong neighbourhood
        if len(nbr[i]) == 0 or agg[i] >= 0 or (agg[nbr[i]] >= 0).any():
            continue
        agg[i] = n_agg
        agg[nbr[i]] = n_agg
        n_agg += 1
    agg1 = agg.copy()
    for i in range(n):  # 2: strongest neighbour aggregated in pass 1, ties to the lowest index
        if agg[i] >= 0 or len(nbr[i]) == 0:
            continue
        ok = agg1[nbr[i]] >= 0
        if ok.any():
            m = np.where(ok, mag[i], -1.0)
            agg[i] = agg1[nbr[i][int(np.argmax(m))]]
    for i in range(n):  # 3: leftovers with their unaggregated strong neighbours
        if agg[i] >= 0 or len(nbr[i]) == 0:
            continue
        agg[i] = n_agg
        free = nbr[i][agg[nbr[i]] < 0]
        agg[free] = n_agg
        n_agg += 1
    return agg, n_agg


def smoothed_prolongation(A, agg, n_agg):
    n = A.shape[0]
    sizes = np.bincount(agg[agg >= 0], minlength=n_agg)
    r = np.nonzero(agg >= 0)[0]
    T = _sorted(sp.csr_matrix((1.0 / np.sqrt(sizes[agg[r]].astype(np.float64)), (r, agg[r])), shape=(n, n_agg)))
    d = A.diagonal()
    rs = _abs_row_sums(A)
    nz = d != 0.0
    lam = float(np.max(rs[nz] / np.abs(d[nz]))) if nz.any() else 0.0
    omega = (4.0 / 3.0) / lam if lam > 0.0 else 0.0
    s = np.zeros(n)
    s[nz] = omega / d[nz]
    AT = _mul(A, T)
    X = AT.copy()
    X.data = s[np.repeat(np.arange(n), np.diff(AT.indptr))] * AT.data
    P = _sorted(T - X)
    P.eliminate_zeros()
    return P


def dense_pseudo_inverse(A):
    """L^-T D^+ L^-1 of A = L D L^T without pivoting; pivots <= PIVOT_TOL * max |a_ii| are dropped with their column."""
    a = np.asarray(A.todense())
    n = a.shape[0]
    tol = PIVOT_TOL * np.max(np.abs(np.diag(a))) if n else 0.0
    L = np.eye(n)
    d = np.zeros(n)
    for k in range(n):
        ld = L[k, :k] * d[:k]
        dk = a[k, k] - L[k, :k] @ ld
        if not dk > tol:
            continue
        d[k] = dk
        L[k + 1:, k] = (a[k + 1:, k] - L[k + 1:, :k] @ ld) / dk
    M = sla.solve_triangular(L, np.eye(n), lower=True, unit_diagonal=True)
    dplus = np.where(d != 0.0, 1.0 / np.where(d != 0.0, d, 1.0), 0.0)
    return M.T @ (dplus[:, None] * M)


class Hierarchy:
    def __init__(self, A, smooth_it=1):
        self.smooth_it = smooth_it
        self.A, self.P, self.R, self.dinv = [], [], [], []
        A = _sorted(A)
        while True:
            self.A.append(A)
            rs = _abs_row_sums(A)
            self.dinv.append(np.where(rs > 0.0, 1.0 / np.where(rs > 0.0, rs, 1.0), 0.0))
            last = A.shape[0] <= COARSE_ROWS or len(self.A) >= MAX_LEVELS
            if not last:
                agg, n_agg = aggregate(A)
                last = n_agg == 0 or n_agg > MAX_KEEP * A.shape[0]
            if last:
                self.Xc = dense_pseudo_inverse(A)
                return
            P = smoothed_prolongation(A, agg, n_agg)
            R = _transpose(P)
            self.P.append(P)
            self.R.append(R)
            A = _mul(R, _mul(A, P))

    @property
    def rows(self):
        return [A.shape[0] for A in self.A]

    @property
    def nnz(self):
        return [A.nnz for A in self.A]

    def _smooth(self, l, b, x):
        A, dinv = self.A[l], self.dinv[l]
        for _ in range(self.smooth_it):
            x = x + dinv * (b - A @ x)
        return x

    def vcycle(self, b, x=None, l=0):
        if l == len(self.A) - 1:
            return self.Xc @ b
        x = np.zeros_like(b) if x is None else x.copy()
        x = self._smooth(l, b, x)
        e = self.vcycle(self.R[l] @ (b - self.A[l] @ x), None, l + 1)
        x = x + self.P[l] @ e
        return self._smooth(l, b, x)


class AMG:
    def __init__(self, A, cycle_it=1, smooth_it=1):
        self.H = Hierarchy(A, smooth_it)
        self.cycle_it = cycle_it

    def mult(self, b, x0=None):
        x = None if x0 is None else x0.copy()
        for _ in range(self.cycle_it):
            x = self.H.vcycle(b, x)
        return x

    __call__ = mult


def nodal_interpolation(G, coords):
    """Pi_c(e, v) = |G(e, v)| t_e[c] / 2 with the edge vectors t = G [x y z] (HYPRE's construction from G and the coordinates)."""
    G = _sorted(G)
    t = G @ np.ascontiguousarray(coords, dtype=np.float64)
    rows = np.repeat(np.arange(G.shape[0]), np.diff(G.indptr))
    Pis = []
    for c in range(3):
        Pi = G.copy()
        Pi.data = 0.5 * np.abs(G.data) * t[rows, c]
        Pis.append(Pi)
    return Pis, t


class AMS:
    """Cycle type 14, "01(3+4+5)10"; `singular` drops the gradient correction."""

    def __init__(self, A, G, coords, cycle_it=1, smooth_it=1, singular=False):
        self.A = _sorted(A)
        self.G = _sorted(G)
        self.Gt = _transpose(self.G)
        self.cycle_it, self.smooth_it, self.singular = cycle_it, smooth_it, singular
        rs = _abs_row_sums(self.A)
        self.dinv = np.where(rs > 0.0, 1.0 / np.where(rs > 0.0, rs, 1.0), 0.0)
        self.Pi, self.t = nodal_interpolation(self.G, coords)
        AG = _mul(self.A, self.G)
        self.HG = None if singular else Hierarchy(_mul(self.Gt, AG), smooth_it)
        self.HPi = [Hierarchy(_mul(_transpose(Pi), _mul(self.A, Pi)), smooth_it) for Pi in self.Pi]

    def hierarchies(self):
        return [self.HG] + self.HPi

    def _smooth(self, b, x):
        for _ in range(self.smooth_it):
            x = x + self.dinv * (b - self.A @ x)
        return x

    def _gradient(self, b, x):
        if self.singular:
            return x
        return x + self.G @ self.HG.vcycle(self.Gt @ (b - self.A @ x))

    def mult(self, b, x0=None):
        x = np.zeros_like(b) if x0 is None else x0.copy()
        for _ in range(self.cycle_it):
            x = self._smooth(b, x)
            x = self._gradient(b, x)
            r = b - self.A @ x
            for Pi, H in zip(self.Pi, self.HPi):
                x = x + Pi @ H.vcycle(Pi.T @ r)
            x = self._gradient(b, x)
            x = self._smooth(b, x)
        return x

    __call__ = mult


def vertex_coords(mesh):
    """Physical vertex coordinates [NV, 3] (the warp applied), indexed like the H1 p = 1 dofs of palace_b200.host.hexspace."""
    xe = mesh.node_coords(1, np.array([0.0, 1.0]))  # [NE, 3, 8], lexicographic corners as mesh.elems
    X = np.zeros((int(mesh.elems.max()) + 1, 3))
    X[mesh.elems.ravel()] = xe.transpose(0, 2, 1).reshape(-1, 3)
    return X

"""CPU: the oracle of the algebraic coarse solvers (oracle/amg.py) on the host layer's spaces.

* Pi_c 1 = G x_c is the Nedelec p = 1 interpolant of the constant field e_c: evaluated through the oracle's basis tables on a
  scrambled, unwarped box (where constants lie in the space) it reproduces e_c, which pins the signs and scale of the global G
  against the ND dofs.
* Growth of the CG iteration count on warped PEC boxes (n^3 elements, solved to 1e-8): AMS on the ND p = 1 K + M and the singular
  AMS on K alone grow by 1.67x and 1.55x from n = 4 to n = 16 (the 1.5x design bound is recorded as an expected failure), while
  Jacobi-PCG on the same K + M grows 7.6x. The H1 matrix at
  n = 4 (125 rows) is below the direct-solve size, so CG + AMG converges there in one iteration; its growth is checked from n = 8,
  the smallest box with a multilevel hierarchy, to n = 16."""
import functools

import numpy as np
import pytest

from oracle import amg
from oracle import pyoracle as O
from oracle import solvers as S
from palace_b200.host import hexspace as hs
from tests import common


@functools.lru_cache(maxsize=None)
def box(n, warp=0.04):
    prob = common.make_problem(n=(n, n, n), p=1, warp=warp, scramble=3, n_attr=3)
    G = common.oracle_interp(prob.h1, prob.nd, hs.discrete_gradient_matrix(1))
    return prob, G, amg.vertex_coords(prob.mesh)


@functools.lru_cache(maxsize=None)
def matrices(n):
    prob, G, X = box(n)
    KM = common.oracle_matrix(prob, O.CURLCURL_MASS, common.coefficient(O.CURLCURL_MASS, 3, "matrix"))
    K = common.oracle_matrix(prob, O.CURLCURL, common.coefficient(O.CURLCURL, 3, "matrix"))
    L = common.oracle_matrix(prob, O.H1_DIFFUSION, common.coefficient(O.H1_DIFFUSION, 3, "matrix"), space=prob.h1)
    return KM, K, L


def _rhs(n_rows, ess, seed):
    b = np.random.default_rng(seed).standard_normal(n_rows)
    b[ess] = 0.0
    return b


@functools.lru_cache(maxsize=None)
def iterations(which, n):
    prob, G, X = box(n)
    KM, K, L = matrices(n)
    if which == "amg":
        b = _rhs(L.shape[0], prob.h1.ess_dofs, 1)
        return S.cg(L, b, amg.AMG(L), rel_tol=1e-8, max_it=2000)[1]
    if which == "ams":
        b = _rhs(KM.shape[0], prob.nd.ess_dofs, 2)
        return S.cg(KM, b, amg.AMS(KM, G, X), rel_tol=1e-8, max_it=2000)[1]
    if which == "jacobi":
        b = _rhs(KM.shape[0], prob.nd.ess_dofs, 2)
        dinv = 1.0 / KM.diagonal()
        return S.cg(KM, b, lambda r: dinv * r, rel_tol=1e-8, max_it=20000)[1]
    assert which == "singular"
    b = K @ _rhs(K.shape[0], prob.nd.ess_dofs, 3)  # in the range of K
    return S.cg(K, b, amg.AMS(K, G, X, singular=True), rel_tol=1e-8, max_it=2000)[1]


@pytest.mark.parametrize("c", [0, 1, 2])
def test_pi_of_ones_is_the_constant_field(c):
    prob, G, X = box(3, warp=0.0)
    Pi, t = amg.nodal_interpolation(G, X)
    u = Pi[c] @ np.ones(G.shape[1])
    assert np.abs(u - G @ X[:, c]).max() < 1e-14
    interp, _, _ = O.nd_hex_tables(1, prob.q1d)  # [3][Q][P] reference basis, native dof order
    idx, ori = prob.nd.native_restriction()
    qd = prob.qdata_ref  # [ne][11][Q]: attribute, w detJ, J^-T column-major
    for e in range(prob.mesh.ne):
        ue = ori[e] * u[idx[e]]
        uref = np.einsum("cqb,b->cq", interp, ue)
        Jit = qd[e, 2:11].reshape(3, 3, -1)  # [col][row][q]
        E = np.einsum("krq,kq->rq", Jit, uref)
        ec = np.zeros((3, 1))
        ec[c] = 1.0
        assert np.abs(E - ec).max() < 1e-12, e


def test_amg_growth():
    it8, it16 = iterations("amg", 8), iterations("amg", 16)
    assert iterations("amg", 4) == 1  # one level: the direct solve
    assert it16 <= 1.5 * it8, (it8, it16)


@pytest.mark.parametrize("which", ["ams", "singular"])
def test_ams_growth(which):
    """Measured: 9, 12, 15 iterations at n = 4, 8, 16 (singular: 11, 14, 17). At n = 4 the auxiliary problems (125 rows) are
    solved directly, so the growth to n = 16 is the price of one V-cycle of the smoothed-aggregation hierarchies."""
    it4, it16 = iterations(which, 4), iterations(which, 16)
    assert it16 <= 1.7 * it4, (which, it4, iterations(which, 8), it16)


@pytest.mark.xfail(strict=True, reason="the 1.5x growth bound is not met yet: 9 -> 15 (K + M) and 11 -> 17 (singular K)")
@pytest.mark.parametrize("which", ["ams", "singular"])
def test_ams_growth_within_one_and_a_half(which):
    assert iterations(which, 16) <= 1.5 * iterations(which, 4)


def test_jacobi_pcg_at_least_doubles():
    it4, it16 = iterations("jacobi", 4), iterations("jacobi", 16)
    assert it16 >= 2 * it4, (it4, it16)
    assert it16 > 1.5 * iterations("ams", 16)


def test_hierarchies_coarsen():
    KM, _, L = matrices(16)
    prob, G, X = box(16)
    s = amg.AMS(KM, G, X)
    for H in s.hierarchies() + [amg.AMG(L).H]:
        assert len(H.rows) >= 2 and H.rows[-1] <= amg.COARSE_ROWS
        assert all(b < amg.MAX_KEEP * a for a, b in zip(H.rows[:-1], H.rows[1:]))


def test_pseudo_inverse_on_a_constant_null_space():
    """The auxiliary gradient matrix G^T A G is singular (G 1 = 0); the dropped pivot makes the coarsest inverse a generalised
    inverse: A X A = A."""
    KM, _, _ = matrices(4)
    prob, G, X = box(4)
    AG = (G.T @ KM @ G).tocsr()
    Xc = amg.dense_pseudo_inverse(AG)
    Ad = AG.toarray()
    assert np.abs(Ad @ Xc @ Ad - Ad).max() < 1e-9 * np.abs(Ad).max()

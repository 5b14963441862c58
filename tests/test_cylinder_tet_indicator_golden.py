"""End-to-end comparison of the flux error estimators on TETRAHEDRA with the reference's own output (CPU, oracle side; slow: runs
only with B2P_SLOW_TESTS=1): error-indicators.csv of
examples/cylinder/waveguide.json -- the periodic tetrahedral waveguide of test_cylinder_tet_golden.py, Nedelec order 4, 15 modes,
grad-flux + curl-flux estimators -- against oracle/estimator.py on the oracle-side tet discretisation: ND_4 with its curl-oriented
transformations, RT_3 (tetspace.build_rt_tet_space), the element-local discrete curl, quadratic geometry.

The global norm agrees to 2.5e-4 with a converged quadrature (conical rules of degree 10 and 12 give 3.003966e-3 and 3.003967e-3; the
reference stores 3.003214e-3, integrating with its degree-8 rule). Unlike eigenvalues (1e-8) an ERROR quantity on curved elements
depends on the rule at this level: the two degree-8 rules of the host layer give 3.003492e-3 (conical) and 2.999598e-3 (43 points,
one negative weight); and the reference's flux projections stop at a relative residual of 1e-6 while the estimated error is 3e-3
of the field, which alone allows 3e-4 in the indicator. On the straight-sided hexahedral cavity, where this repository integrates with the reference's own rule, the
same pipeline reproduces the stored norm to 1e-7 (tests/test_cylinder_indicator_golden.py)."""
import os

import numpy as np
import pytest
import scipy.sparse.linalg as spla

from oracle import estimator as E
from oracle import pyoracle as O
from palace_b200.host import tetspace as ts
from tests import common
from tests.test_cylinder_tet_golden import FIX, oracle_matrix, sigma_target, space_and_tables
from tests.test_zzflux_curl_oriented_gpu import assembled, dense_T

REF_NORM, REF_MEAN = 3.003213590936e-03, 1.587572734952e-04   # test/data/regression/ref/cylinder/waveguide/error-indicators.csv


@pytest.mark.skipif(os.environ.get("B2P_SLOW_TESTS") != "1", reason="about a minute of NumPy loops: B2P_SLOW_TESTS=1")
def test_tet_waveguide_error_indicators_against_the_reference():
    p = int(FIX["order"])
    mesh, nd, interp, curl, qd = space_and_tables(p)                       # conical rule of degree 2p + 2
    _, _, qpts, _ = ts.nd_tet_tables(p, 2 * p + 2)
    rt = ts.build_rt_tet_space(mesh, nd, p - 1)
    rt_i = ts.rt_tet_element(p - 1).tabulate(qpts)
    ne, eps = mesh.ne, float(FIX["eps_r"])
    K, M = oracle_matrix(nd, O.CURLCURL, interp, curl, qd), oracle_matrix(nd, O.ND_MASS, interp, curl, qd)
    free = np.setdiff1d(np.arange(nd.ndofs), nd.ess_dofs)
    lam, V = common.eigsh_above(K[free][:, free].tocsc(), M[free][:, free].tocsc(), 15, sigma_target(), vectors=True)
    I3 = [np.eye(3)] * ne
    co_r = np.zeros((ne, rt.P, 3), dtype=np.int8)
    co_r[:, :, 1] = rt.orient
    Mrt = assembled(qd, rt_i, E.HDIV, rt.idx, co_r, rt.ndofs, rt_i, E.HDIV, rt.idx, co_r, rt.ndofs, I3)
    F = assembled(qd, interp, E.HCURL, nd.idx, nd.curl_orient, nd.ndofs, rt_i, E.HDIV, rt.idx, co_r, rt.ndofs, I3)
    lu_rt, lu_nd = spla.splu(Mrt.tocsc()), spla.splu(M.tocsc())
    C = ts.tet_discrete_curl(p)
    Tn = [dense_T(nd.curl_orient[e]) for e in range(ne)]
    dr, dn = np.arange(ne * rt.P).reshape(ne, rt.P), np.arange(ne * nd.P).reshape(ne, nd.P)
    onr, onn = np.ones((ne, rt.P)), np.ones((ne, nd.P))
    se, ise = [np.sqrt(eps) * np.eye(3)] * ne, [np.eye(3) / np.sqrt(eps)] * ne
    acc = np.zeros(ne)
    for j in range(15):
        v = np.zeros(nd.ndofs)
        v[free] = V[:, j]
        B = np.zeros(rt.ndofs)
        for e in range(ne):
            B[rt.idx[e]] = rt.orient[e] * (C @ (Tn[e] @ v[nd.idx[e]]))
        B /= np.sqrt(lam[j] / eps)
        Eel, Emag = 0.5 * eps * (v @ (M @ v)), 0.5 * (B @ (Mrt @ B))
        assert abs(Eel / Emag - 1) < 1e-10                                  # discrete curl, RT mass and the pencil are consistent
        D, H = lu_rt.solve(eps * (F @ v)), lu_nd.solve(F.T @ B)
        ve = np.concatenate([Tn[e] @ v[nd.idx[e]] for e in range(ne)])
        He = np.concatenate([Tn[e] @ H[nd.idx[e]] for e in range(ne)])
        Be = np.concatenate([rt.orient[e] * B[rt.idx[e]] for e in range(ne)])
        De = np.concatenate([rt.orient[e] * D[rt.idx[e]] for e in range(ne)])
        eg = E.element_errors(qd, interp, E.HCURL, dn, onn, ve, se, rt_i, E.HDIV, dr, onr, De, ise)
        ec = E.element_errors(qd, rt_i, E.HDIV, dr, onr, Be, I3, interp, E.HCURL, dn, onn, He, I3)
        acc += 0.5 / (Eel + Emag) * (eg + ec)
    e_ = np.sqrt(acc / 15)
    print("Norm, Min, Max, Mean:", np.linalg.norm(e_), e_.min(), e_.max(), e_.mean(), " reference norm / mean:", REF_NORM, REF_MEAN)
    assert abs(np.linalg.norm(e_) / REF_NORM - 1) < 5e-4 and abs(e_.mean() / REF_MEAN - 1) < 1e-3

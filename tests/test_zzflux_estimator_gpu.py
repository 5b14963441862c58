"""CurlFluxErrorEstimator (/root/reference/palace/linalg/errorestimator.cpp:112-270,400-513) through the C ABI against the NumPy
restatement of oracle/estimator.py: mixed H(div) -> H(curl) mass operator, flux projection (PCG + damped Jacobi on the ND mass
matrix), element-wise error integrals, complex fields, the final square root and scaling. The discontinuous flux is B = curl E
in the Raviart-Thomas space RT_{p-1} (host layer: build_rt_space, discrete_curl_matrix). The oracle evaluates the bases from its
own tables; the library gets the host layer's tables, so the two sides share only the dof numbering."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

from oracle import estimator as E
from oracle import pyoracle as O
from palace_b200.host import coeff as cf
from palace_b200.host import hexspace as hs
from tests import common

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def curl_dofs(nd, rt, x):
    """B = Curl E: global RT dofs of the discrete curl of the ND field x."""
    Cl = hs.discrete_curl_matrix(nd.p)
    B = np.zeros(rt.ndofs)
    for e in range(nd.lex_gid.shape[0]):
        B[rt.lex_gid[e]] = rt.lex_sign[e] * (Cl @ (nd.lex_sign[e] * x[nd.lex_gid[e]]))
    return B


@pytest.fixture(scope="module", params=[(2, 0.04), (3, 0.0)])
def setup(request, b2p_ctx):
    from palace_b200 import capi

    p, warp = request.param
    n_attr = 3
    prob = common.make_problem(n=(3, 2, 2), p=p, warp=warp, n_attr=n_attr)
    geom = common.gpu_geom(b2p_ctx, prob)
    nd = prob.nd
    rt = hs.build_rt_space(prob.mesh, prob.topo, p)
    # mu^-1 per attribute: the striped symmetric positive definite matrices of the reference unit tests
    am, mc = cf.test_suite_coefficient(n_attr, "matrix")
    muinv = np.stack([mc[am[a]] for a in range(n_attr)])
    c_flux = np.stack([m.ravel(order="F") for m in muinv])
    c_disc = np.stack([E.spd_power(m, 0.5).ravel(order="F") for m in muinv])
    c_smooth = np.stack([E.spd_power(m, -0.5).ravel(order="F") for m in muinv])
    # library side: host-layer tables (lexicographic ND and RT bases), ND mass without coefficient and without essential dofs
    ones = np.ones_like(nd.lex_sign)
    sp_rt = dict(P=rt.P, map_type=capi.MAP_HDIV, interp=hs.rt_hex_dense_interp(p, prob.q1d), idx=rt.lex_gid, orient=rt.lex_sign, lsize=rt.ndofs)
    sp_nd = dict(P=nd.P, map_type=capi.MAP_HCURL, interp=hs.nd_hex_dense_interp(p, prob.q1d), idx=nd.lex_gid, orient=nd.lex_sign, lsize=nd.ndofs)
    blob1 = cf.coeff_ctx(a=1.0)
    mop = common.gpu_op(b2p_ctx, geom, prob, O.ND_MASS, blob1)
    Mnd = capi.Operator.par(b2p_ctx, nd.ndofs, nd.ndofs, [mop], None, None, diag_policy=1)
    est = capi.FluxEstimator(b2p_ctx, geom, sp_rt, sp_nd, c_flux, c_disc, c_smooth, Mnd, tol=1e-13, max_it=2000)
    # oracle side: its own tables (ND in native order with the native restriction, RT from the oracle's 1-D bases)
    nd_interp, _, _ = O.nd_hex_tables(p, prob.q1d)
    idx_n, ori_n = nd.native_restriction()
    rt_interp = E.rt_hex_tables(p, prob.q1d)
    attr = prob.mesh.attr - 1
    celem = lambda tab: [E._mat33(tab[a]) for a in attr]
    o = dict(qd=prob.qdata_ref, nd_interp=nd_interp, idx_n=idx_n.astype(np.int64), ori_n=ori_n.astype(float), rt_interp=rt_interp,
             idx_r=rt.lex_gid, ori_r=rt.lex_sign.astype(float), c_flux=celem(c_flux), c_disc=celem(c_disc), c_smooth=celem(c_smooth))
    o["F"] = E.mixed_mass_matrix(o["qd"], rt_interp, E.HDIV, o["idx_r"], o["ori_r"], rt.ndofs, nd_interp, E.HCURL, o["idx_n"], o["ori_n"],
                                 nd.ndofs, o["c_flux"])
    o["M"] = common.oracle_matrix(prob, O.ND_MASS, blob1, space=nd, eliminate=False)
    del ones
    return dict(p=p, warp=warp, prob=prob, nd=nd, rt=rt, est=est, o=o, keep=[mop, Mnd, geom])


def oracle_estimates(s, B):
    o = s["o"]
    H = spla.spsolve(o["M"].tocsc(), o["F"] @ B)
    eta2 = E.element_errors(o["qd"], o["rt_interp"], E.HDIV, o["idx_r"], o["ori_r"], B, o["c_disc"], o["nd_interp"], E.HCURL, o["idx_n"],
                            o["ori_n"], H, o["c_smooth"])
    return H, eta2


def test_projection_and_element_errors_match_the_oracle(b2p_ctx, setup):
    s = setup
    rng = np.random.default_rng(51)
    B = curl_dofs(s["nd"], s["rt"], rng.standard_normal(s["nd"].ndofs))
    H_ref, eta2_ref = oracle_estimates(s, B)
    Hd = torch.zeros(s["nd"].ndofs, dtype=torch.float64, device="cuda")
    s["est"].project(_dev(B), Hd)
    st = s["est"].stats()
    assert st["converged"]
    assert _rel(Hd.cpu().numpy(), H_ref) < 1e-10
    ne = s["prob"].mesh.ne
    ed = torch.zeros(ne, dtype=torch.float64, device="cuda")
    s["est"].integrate(_dev(B), Hd, ed)
    assert _rel(ed.cpu().numpy(), eta2_ref) < 1e-9
    s["est"].integrate(_dev(B), Hd, ed)  # accumulates (the second part of a complex field)
    assert _rel(ed.cpu().numpy(), 2.0 * eta2_ref) < 1e-9


@pytest.mark.parametrize("Et", [0.0, 3.7])
def test_indicator_of_real_and_complex_fields(b2p_ctx, setup, Et):
    """AddErrorIndicator: eta_K = sqrt(s (eta_K^2(Re) + eta_K^2(Im))), s = 0.5 / Et or 1."""
    s = setup
    rng = np.random.default_rng(53)
    Br = curl_dofs(s["nd"], s["rt"], rng.standard_normal(s["nd"].ndofs))
    Bi = curl_dofs(s["nd"], s["rt"], 0.3 * rng.standard_normal(s["nd"].ndofs))
    _, e2r = oracle_estimates(s, Br)
    _, e2i = oracle_estimates(s, Bi)
    scale = 0.5 / Et if Et > 0.0 else 1.0
    ne = s["prob"].mesh.ne
    ed = torch.full((ne,), 7.0, dtype=torch.float64, device="cuda")  # overwritten, not accumulated
    s["est"].indicator(_dev(Br), None, Et, ed)
    assert _rel(ed.cpu().numpy(), np.sqrt(scale * e2r)) < 1e-9
    s["est"].indicator(_dev(Br), _dev(Bi), Et, ed)
    assert _rel(ed.cpu().numpy(), np.sqrt(scale * (e2r + e2i))) < 1e-9


def test_smooth_flux_has_no_error_on_an_affine_mesh(b2p_ctx, setup):
    """A constant B on straight elements with mu = 1 everywhere would be reproduced exactly; with the striped mu^-1 the flux
    mu^-1 B jumps across material interfaces, so only the estimate of a field whose flux IS in the ND space vanishes: take
    mu^-1 B = const inside one material. Simplest exact case: all elements of the mesh carry the SAME material. A warped setup
    runs the check at its order on the same mesh without the warp."""
    from palace_b200 import capi

    s = setup
    prob, nd, rt, p = s["prob"], s["nd"], s["rt"], s["p"]
    geom, Mnd = s["keep"][2], s["keep"][1]
    if s["warp"] != 0.0:
        # a constant field is in the RT space only on straight-sided elements: the same order on the unwarped mesh
        prob = common.make_problem(n=(3, 2, 2), p=p, warp=0.0, n_attr=3)
        geom = common.gpu_geom(b2p_ctx, prob)
        nd, rt = prob.nd, hs.build_rt_space(prob.mesh, prob.topo, p)
        mop = common.gpu_op(b2p_ctx, geom, prob, O.ND_MASS, cf.coeff_ctx(a=1.0))
        Mnd = capi.Operator.par(b2p_ctx, nd.ndofs, nd.ndofs, [mop], None, None, diag_policy=1)
    # estimator with one material: identity mu^-1
    eye = np.eye(3).ravel()[None, :].repeat(3, axis=0)
    sp_rt = dict(P=rt.P, map_type=capi.MAP_HDIV, interp=hs.rt_hex_dense_interp(p, prob.q1d), idx=rt.lex_gid, orient=rt.lex_sign, lsize=rt.ndofs)
    sp_nd = dict(P=nd.P, map_type=capi.MAP_HCURL, interp=hs.nd_hex_dense_interp(p, prob.q1d), idx=nd.lex_gid, orient=nd.lex_sign, lsize=nd.ndofs)
    est = capi.FluxEstimator(b2p_ctx, geom, sp_rt, sp_nd, eye, eye, eye, Mnd, tol=1e-13, max_it=2000)
    # RT dofs of the constant field c: reference components u^ = detJ J^-1 c on every (affine) element
    c = np.array([0.3, -1.1, 0.7])
    B = np.zeros(rt.ndofs)
    lay = hs._rt_lex_layout(p)
    comp = np.array([l[0] for l in lay])
    for e in range(prob.mesh.ne):
        A = E._mat33(prob.qdata_ref[e, 2:, 0])          # J^-T (constant on the element)
        uhat = (A.T @ c) / np.linalg.det(A)              # detJ J^-1 c
        B[rt.lex_gid[e]] = rt.lex_sign[e] * uhat[comp]
    ed = torch.zeros(prob.mesh.ne, dtype=torch.float64, device="cuda")
    est.indicator(_dev(B), None, 0.0, ed)
    vol = prob.qdata_ref[:, 1, :].sum(axis=1)
    assert (ed.cpu().numpy() < 1e-9 * np.sqrt(vol * (c @ c))).all()


def test_table_described_mass_operator_and_grad_flux_configuration(b2p_ctx, setup):
    """b2p_operator_vecfe_mass on the Raviart-Thomas space (Mult, diagonal) against the oracle matrix, and the estimator with the
    roles of GradFluxErrorEstimator (errorestimator.cpp:272-398): discontinuous flux eps E with E in the ND space, smooth flux D in
    the RT space, M = RT mass matrix, integrand |eps^(-1/2) D - eps^(1/2) E|^2 (f_apply_hcurlhdiv_error_33)."""
    from palace_b200 import capi

    s = setup
    prob, nd, rt, p, o = s["prob"], s["nd"], s["rt"], s["p"], s["o"]
    geom = s["keep"][2]
    sp_rt = dict(P=rt.P, map_type=capi.MAP_HDIV, interp=hs.rt_hex_dense_interp(p, prob.q1d), idx=rt.lex_gid, orient=rt.lex_sign, lsize=rt.ndofs)
    sp_nd = dict(P=nd.P, map_type=capi.MAP_HCURL, interp=hs.nd_hex_dense_interp(p, prob.q1d), idx=nd.lex_gid, orient=nd.lex_sign, lsize=nd.ndofs)
    Mrt = capi.vecfe_mass_operator(b2p_ctx, geom, sp_rt)
    ident = [np.eye(3)] * prob.mesh.ne
    Mo = E.mixed_mass_matrix(o["qd"], o["rt_interp"], E.HDIV, o["idx_r"], o["ori_r"], rt.ndofs, o["rt_interp"], E.HDIV, o["idx_r"], o["ori_r"],
                             rt.ndofs, ident)
    rng = np.random.default_rng(57)
    x = rng.standard_normal(rt.ndofs)
    yd = torch.empty(rt.ndofs, dtype=torch.float64, device="cuda")
    Mrt.mult(_dev(x), yd)
    assert _rel(yd.cpu().numpy(), Mo @ x) < 1e-12
    dd = torch.empty(rt.ndofs, dtype=torch.float64, device="cuda")
    Mrt.assemble_diagonal(dd)
    assert _rel(dd.cpu().numpy(), Mo.diagonal()) < 1e-12
    # the same operator with a coefficient table agrees with the oracle's coefficient version
    n_attr = 3
    am, mc = cf.test_suite_coefficient(n_attr, "matrix")
    eps = np.stack([mc[am[a]] for a in range(n_attr)])
    c_eps = np.stack([m.ravel(order="F") for m in eps])
    attr = prob.mesh.attr - 1
    Mo_eps = E.mixed_mass_matrix(o["qd"], o["rt_interp"], E.HDIV, o["idx_r"], o["ori_r"], rt.ndofs, o["rt_interp"], E.HDIV, o["idx_r"], o["ori_r"],
                                 rt.ndofs, [E._mat33(c_eps[a]) for a in attr])
    Mrt_eps = capi.vecfe_mass_operator(b2p_ctx, geom, sp_rt, c_eps)
    Mrt_eps.mult(_dev(x), yd)
    assert _rel(yd.cpu().numpy(), Mo_eps @ x) < 1e-12
    # GradFlux roles: flux space ND with eps, smooth space RT
    c_disc = np.stack([E.spd_power(m, 0.5).ravel(order="F") for m in eps])
    c_smooth = np.stack([E.spd_power(m, -0.5).ravel(order="F") for m in eps])
    est = capi.FluxEstimator(b2p_ctx, geom, sp_nd, sp_rt, c_eps, c_disc, c_smooth, Mrt, tol=1e-13, max_it=4000)
    Ev = rng.standard_normal(nd.ndofs)
    celem = lambda tab: [E._mat33(tab[a]) for a in attr]
    F = E.mixed_mass_matrix(o["qd"], o["nd_interp"], E.HCURL, o["idx_n"], o["ori_n"], nd.ndofs, o["rt_interp"], E.HDIV, o["idx_r"], o["ori_r"],
                            rt.ndofs, celem(c_eps))
    D_ref = spla.spsolve(Mo.tocsc(), F @ Ev)
    eta2 = E.element_errors(o["qd"], o["nd_interp"], E.HCURL, o["idx_n"], o["ori_n"], Ev, celem(c_disc), o["rt_interp"], E.HDIV, o["idx_r"],
                            o["ori_r"], D_ref, celem(c_smooth))
    Dd = torch.zeros(rt.ndofs, dtype=torch.float64, device="cuda")
    est.project(_dev(Ev), Dd)
    assert est.stats()["converged"]
    assert _rel(Dd.cpu().numpy(), D_ref) < 1e-9
    ed = torch.zeros(prob.mesh.ne, dtype=torch.float64, device="cuda")
    est.integrate(_dev(Ev), Dd, ed)
    assert _rel(ed.cpu().numpy(), eta2) < 1e-8
    # TimeDependentFluxErrorEstimator: both flux terms in one array, then one square root
    B = curl_dofs(nd, rt, rng.standard_normal(nd.ndofs))
    Hd = torch.zeros(nd.ndofs, dtype=torch.float64, device="cuda")
    s["est"].project(_dev(B), Hd)
    s["est"].integrate(_dev(B), Hd, ed)
    _, e2c = oracle_estimates(s, B)
    capi.flux_sqrt_scale(b2p_ctx, prob.mesh.ne, 0.25, ed)
    assert _rel(ed.cpu().numpy(), np.sqrt(0.25 * (eta2 + e2c))) < 1e-8


def test_argument_checks(b2p_ctx, setup):
    from palace_b200 import capi

    s = setup
    prob, nd, rt, p = s["prob"], s["nd"], s["rt"], s["p"]
    eye = np.eye(3).ravel()[None, :]
    sp_rt = dict(P=rt.P, map_type=capi.MAP_HDIV, interp=hs.rt_hex_dense_interp(p, prob.q1d), idx=rt.lex_gid, orient=rt.lex_sign, lsize=rt.ndofs)
    sp_nd = dict(P=nd.P, map_type=capi.MAP_HCURL, interp=hs.nd_hex_dense_interp(p, prob.q1d), idx=nd.lex_gid, orient=nd.lex_sign, lsize=nd.ndofs)
    with pytest.raises(capi.B2PError, match="attribute"):
        capi.FluxEstimator(b2p_ctx, s["keep"][2], sp_rt, sp_nd, eye, eye, eye, s["keep"][1])  # 3 attributes on the mesh, 1 in the tables
    bad = dict(sp_nd, map_type=7)
    with pytest.raises(capi.B2PError, match="map type"):
        capi.FluxEstimator(b2p_ctx, s["keep"][2], sp_rt, bad, eye.repeat(3, axis=0), eye.repeat(3, axis=0), eye.repeat(3, axis=0), s["keep"][1])

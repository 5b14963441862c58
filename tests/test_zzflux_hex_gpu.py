"""GPU: the flux estimator on hexahedra with sum-factorised spaces (b2p_flux_estimator_create_hex, b2p_hex_flux.cu) against the
oracle's mixed mass matrix and element errors and against the dense-table estimator (b2p_flux_estimator_create): Flux in both
directions with non-symmetric coefficients, the error integrals of the curl-flux and grad-flux configurations, projection and
indicator under Jacobi and multigrid, the cylinder cavity end to end, and the refusals. Meshes are warped, with scrambled element
frames and 3 attributes; their 9 elements leave a partly filled last batch for every production batch size (8, 4, 2, 2, 1)."""
import os

import numpy as np
import pytest

from oracle import estimator as E
from oracle import pyoracle as O
from palace_b200.host import assemble as asm
from palace_b200.host import coeff as cf
from palace_b200.host import hexmesh as hm
from palace_b200.host import hexspace as hs
from tests import common
from tests.test_cylinder_golden import FIX
from tests.test_cylinder_indicator_golden import REF_NORM, cavity_modes, curl_dofs, oracle_indicators

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

_rng = np.random.default_rng(11)
# non-symmetric per-attribute flux coefficients (column-major), and symmetric positive definite tensors with their square roots
NONSYM = np.stack([(rng_m + 3.0 * np.eye(3)).ravel(order="F") for rng_m in _rng.standard_normal((3, 3, 3))])
_G = _rng.standard_normal((3, 3, 3))
SPD = np.einsum("kij,klj->kil", _G, _G) + 2.0 * np.eye(3)[None]
SPD_FLUX = np.stack([m.ravel(order="F") for m in SPD])
SPD_DISC = np.stack([E.spd_power(m, 0.5).ravel(order="F") for m in SPD])
SPD_SMOOTH = np.stack([E.spd_power(m, -0.5).ravel(order="F") for m in SPD])


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return np.linalg.norm(a - b) / np.linalg.norm(b)


class Case:
    """One mesh at (p, q1d) with the ND and RT spaces described three ways: b2p_op_desc fields (the tensor estimator), dense tables
    (the dense estimator) and the oracle's own tables."""

    def __init__(self, ctx, p, q1d, n=(3, 3, 1)):
        from palace_b200 import capi

        mesh = hm.box_mesh(n, (1.0, 0.7, 0.9), warp_amp=0.04, scramble_seed=3, n_attr=3)
        self.ctx, self.p, self.q1d, self.mesh = ctx, p, q1d, mesh
        self.prob = common.problem_on_mesh(mesh, p=p, q1d=q1d)
        nd, rt = self.prob.nd, hs.build_rt_space(mesh, self.prob.topo, p)
        self.nd, self.rt = nd, rt
        self.geom = common.gpu_geom(ctx, self.prob)
        t = hs.tables_1d(p, q1d)
        idx, ori = nd.native_restriction()
        self.hex = {"nd": dict(kind=capi.ND_MASS, p=p, lsize=nd.ndofs, idx=idx, orient=ori, dof_map=nd.dof_map, Bo=t.Bo, Bc=t.Bc),
                    "rt": dict(kind=capi.RT_MASS, p=p, lsize=rt.ndofs, idx=rt.lex_gid, orient=rt.lex_sign, Bo=t.Bo, Bc=t.Bc)}
        self.dense = {"nd": dict(P=nd.P, map_type=capi.MAP_HCURL, interp=hs.nd_hex_dense_interp(p, q1d), idx=nd.lex_gid, orient=nd.lex_sign,
                                 lsize=nd.ndofs),
                      "rt": dict(P=rt.P, map_type=capi.MAP_HDIV, interp=hs.rt_hex_dense_interp(p, q1d), idx=rt.lex_gid, orient=rt.lex_sign,
                                 lsize=rt.ndofs)}
        self.n = {"nd": nd.ndofs, "rt": rt.ndofs}
        self.mop = capi.Op.create(ctx, self.geom, capi.ND_MASS, p, nd.ndofs, idx, ori, nd.dof_map, t.Bo, t.Bc, t.Gc, cf.coeff_ctx(a=1.0))
        self.rop = capi.Op.create(ctx, self.geom, capi.RT_MASS, p, rt.ndofs, rt.lex_gid, rt.lex_sign, None, t.Bo, t.Bc, None,
                                  cf.coeff_ctx(a=1.0))
        self.M = {"nd": capi.Operator.par(ctx, nd.ndofs, nd.ndofs, [self.mop]), "rt": capi.Operator.par(ctx, rt.ndofs, rt.ndofs, [self.rop])}
        nd_interp, _, _ = O.nd_hex_tables(p, q1d)
        self.o = {"nd": (nd_interp, E.HCURL, idx.astype(np.int64), ori.astype(float), nd.ndofs),
                  "rt": (E.rt_hex_tables(p, q1d), E.HDIV, rt.lex_gid, rt.lex_sign.astype(float), rt.ndofs)}
        self.attr = mesh.attr - 1

    def celem(self, tab):
        return [E._mat33(tab[a]) for a in self.attr]

    def oracle_flux(self, flux, coef):
        smooth = "rt" if flux == "nd" else "nd"
        return E.mixed_mass_matrix(self.prob.qdata_ref, *self.o[flux], *self.o[smooth], self.celem(coef))

    def oracle_errors(self, flux, x1, x2, c1, c2):
        smooth = "rt" if flux == "nd" else "nd"
        i1, m1, g1, s1, _ = self.o[flux]
        i2, m2, g2, s2, _ = self.o[smooth]
        return E.element_errors(self.prob.qdata_ref, i1, m1, g1, s1, x1, self.celem(c1), i2, m2, g2, s2, x2, self.celem(c2))

    def estimators(self, flux, cfl, cd, cs, tol=1e-13, max_it=4000):
        """(tensor, dense) estimators with `flux` ("nd" or "rt") as the flux space and the other as the smooth space."""
        from palace_b200 import capi

        smooth = "rt" if flux == "nd" else "nd"
        M = self.M[smooth]
        th = capi.FluxEstimator.hex(self.ctx, self.geom, self.hex[flux], self.hex[smooth], cfl, cd, cs, M, tol=tol, max_it=max_it)
        td = capi.FluxEstimator(self.ctx, self.geom, self.dense[flux], self.dense[smooth], cfl, cd, cs, M, tol=tol, max_it=max_it)
        return th, td


_cases = {}


def case(ctx, p, q1d):
    """The Case at (p, q1d), built once per module (9 elements: small on host and device)."""
    if (p, q1d) not in _cases:
        _cases[(p, q1d)] = Case(ctx, p, q1d)
    return _cases[(p, q1d)]


PQ = [(p, q) for p in range(1, 7) for q in (p + 1, p + 2) if q <= 7]


def expected_kernel(what, p, q1d):
    """The route: the production kernel at q1d = p + 1 for p >= 2 (the host layer's tables are mirror-symmetric), the cross-check
    kernel otherwise."""
    return f"flux_hex_{what}7_kernel" if q1d == p + 1 and p >= 2 else f"flux_hex_{what}_kernel"


@pytest.mark.parametrize("p,q1d", PQ)
@pytest.mark.parametrize("flux", ["nd", "rt"])
def test_flux_mult_matches_the_oracle_and_the_dense_estimator(b2p_ctx, p, q1d, flux):
    from palace_b200 import capi

    c = case(b2p_ctx, p, q1d)
    smooth = "rt" if flux == "nd" else "nd"
    th, td = c.estimators(flux, NONSYM, NONSYM, NONSYM)
    x = np.random.default_rng(p + 10 * q1d).standard_normal(c.n[flux])
    y = torch.full((c.n[smooth],), np.nan, dtype=torch.float64, device="cuda")  # overwritten, not accumulated
    th.flux_mult(_dev(x), y)
    assert capi.last_launch(b2p_ctx)["kernel"] == expected_kernel("mixed", p, q1d)
    y = y.cpu().numpy()
    y_ref = c.oracle_flux(flux, NONSYM) @ x
    assert _rel(y, y_ref) < 1e-12
    yd = torch.zeros(c.n[smooth], dtype=torch.float64, device="cuda")
    td.flux_mult(_dev(x), yd)
    assert _rel(y, yd.cpu().numpy()) < 1e-12


INTEGRATE_PQ = [(1, 2), (2, 3), (2, 4), (3, 4), (4, 5), (4, 6), (5, 6), (6, 7)]


@pytest.mark.parametrize("p,q1d", INTEGRATE_PQ)
@pytest.mark.parametrize("flux", ["rt", "nd"])  # curl-flux (flux RT, smooth ND) and grad-flux (flux ND, smooth RT)
def test_integrate_matches_the_oracle_and_is_reproducible(b2p_ctx, p, q1d, flux):
    from palace_b200 import capi

    c = case(b2p_ctx, p, q1d)
    smooth = "rt" if flux == "nd" else "nd"
    th, td = c.estimators(flux, SPD_FLUX, SPD_DISC, SPD_SMOOTH)
    rng = np.random.default_rng(3 * p + q1d)
    x1, x2 = rng.standard_normal(c.n[flux]), rng.standard_normal(c.n[smooth])
    eta2 = c.oracle_errors(flux, x1, x2, SPD_DISC, SPD_SMOOTH)
    ne = c.mesh.ne
    start = np.linspace(0.5, 1.5, ne)
    runs = []
    for _ in range(2):
        est = _dev(start)
        th.integrate(_dev(x1), _dev(x2), est)
        assert capi.last_launch(b2p_ctx)["kernel"] == expected_kernel("error", p, q1d)
        runs.append(est.cpu().numpy())
    assert np.array_equal(runs[0], runs[1])  # bit for bit
    assert _rel(runs[0] - start, eta2) < 1e-12  # accumulated onto the non-zero start
    ed = _dev(start)
    td.integrate(_dev(x1), _dev(x2), ed)
    assert _rel(runs[0] - start, ed.cpu().numpy() - start) < 1e-12


def _levels(c, space, orders):
    """Operators (coarse -> fine, ending on the case's mass operator) and prolongations of the p-hierarchy of `space`."""
    from palace_b200 import capi

    mesh, topo = c.mesh, c.prob.topo
    if space == "rt":
        spaces = [hs.build_rt_space(mesh, topo, q) for q in orders[:-1]] + [c.rt]
        ops = [capi.Operator.par(c.ctx, s.ndofs, s.ndofs, [c.rop.coarsen(s.p, s.ndofs, s.lex_gid, s.lex_sign, None, hs.tables_1d(s.p, c.q1d).Bo,
                                                                         hs.tables_1d(s.p, c.q1d).Bc, None)]) for s in spaces[:-1]]
        comps = asm.rt_prolongation_comps
    else:
        spaces = [hs.build_nd_space(mesh, topo, q) for q in orders[:-1]] + [c.nd]
        ops = []
        for s in spaces[:-1]:
            idx, ori = s.native_restriction()
            tt = hs.tables_1d(s.p, c.q1d)
            ops.append(capi.Operator.par(c.ctx, s.ndofs, s.ndofs, [c.mop.coarsen(s.p, s.ndofs, idx, ori, s.dof_map, tt.Bo, tt.Bc, tt.Gc)]))
        comps = asm.nd_prolongation_comps
    P = [common.gpu_interp(c.ctx, a, b, comps(x, y)) for a, b, x, y in zip(spaces[:-1], spaces[1:], orders[:-1], orders[1:])]
    return ops + [c.M[space]], P


@pytest.mark.parametrize("p,q1d", [(3, 4), (2, 4)])
@pytest.mark.parametrize("flux", ["rt", "nd"])
@pytest.mark.parametrize("solver", ["jacobi", "multigrid"])
def test_project_and_indicator_equal_the_dense_estimator(b2p_ctx, p, q1d, flux, solver):
    c = case(b2p_ctx, p, q1d)
    smooth = "rt" if flux == "nd" else "nd"
    th, td = c.estimators(flux, SPD_FLUX, SPD_DISC, SPD_SMOOTH)
    if solver == "multigrid":
        for est in (th, td):
            ops, P = _levels(c, smooth, asm.p_sequence(p))
            est.set_multigrid(ops, P, coarse_type=1, coarse_tol=1e-10, coarse_max_it=2000)
    rng = np.random.default_rng(5 * p + q1d)
    if flux == "rt":
        xr, xi = curl_dofs(c.nd, c.rt, rng.standard_normal(c.nd.ndofs)), curl_dofs(c.nd, c.rt, 0.3 * rng.standard_normal(c.nd.ndofs))
    else:
        xr, xi = rng.standard_normal(c.nd.ndofs), 0.3 * rng.standard_normal(c.nd.ndofs)
    out = {}
    for name, est in (("hex", th), ("dense", td)):
        H = torch.zeros(c.n[smooth], dtype=torch.float64, device="cuda")
        est.project(_dev(xr), H)
        assert est.stats()["converged"]
        e1 = torch.full((c.mesh.ne,), 7.0, dtype=torch.float64, device="cuda")
        est.indicator(_dev(xr), None, 0.0, e1)
        e2 = torch.zeros(c.mesh.ne, dtype=torch.float64, device="cuda")
        est.indicator(_dev(xr), _dev(xi), 3.7, e2)
        out[name] = [H.cpu().numpy(), e1.cpu().numpy(), e2.cpu().numpy()]
    for a, b in zip(out["hex"], out["dense"]):
        assert _rel(a, b) < 1e-10


def test_cylinder_estimators_on_the_tensor_path(b2p_ctx):
    from palace_b200 import capi

    p = int(os.environ.get("B2P_TEST_ORDER", int(FIX["order"])))  # (B2P_TEST_ORDER=2: a quick run, no comparison with the stored norm)
    c = cavity_modes(p)
    mesh, topo, nd, rt, q1d, eps = c["mesh"], c["topo"], c["nd"], c["rt"], c["q1d"], c["eps"]
    ne = mesh.ne
    geom = capi.Geom.from_qdata(b2p_ctx, c["qd"], q1d)
    t = hs.tables_1d(p, q1d)
    mop = capi.Op.create(b2p_ctx, geom, capi.ND_MASS, p, nd.ndofs, c["idx"], c["ori"], nd.dof_map, t.Bo, t.Bc, t.Gc, cf.coeff_ctx(a=1.0))
    rop = capi.Op.create(b2p_ctx, geom, capi.RT_MASS, p, rt.ndofs, rt.lex_gid, rt.lex_sign, None, t.Bo, t.Bc, None, cf.coeff_ctx(a=1.0))
    Mnd = capi.Operator.par(b2p_ctx, nd.ndofs, nd.ndofs, [mop])
    Mrt = capi.Operator.par(b2p_ctx, rt.ndofs, rt.ndofs, [rop])
    sp_nd = dict(kind=capi.ND_MASS, p=p, lsize=nd.ndofs, idx=c["idx"], orient=c["ori"], dof_map=nd.dof_map, Bo=t.Bo, Bc=t.Bc)
    sp_rt = dict(kind=capi.RT_MASS, p=p, lsize=rt.ndofs, idx=rt.lex_gid, orient=rt.lex_sign, Bo=t.Bo, Bc=t.Bc)
    I9 = np.eye(3).ravel()[None]
    curl_est = capi.FluxEstimator.hex(b2p_ctx, geom, sp_rt, sp_nd, I9, I9, I9, Mnd, tol=1e-12, max_it=20000)
    grad_est = capi.FluxEstimator.hex(b2p_ctx, geom, sp_nd, sp_rt, eps * I9, np.sqrt(eps) * I9, I9 / np.sqrt(eps), Mrt, tol=1e-12,
                                      max_it=20000)
    orders = asm.p_sequence(p)

    def levels(fine, build, coarsen, comps):
        spaces = [build(q) for q in orders[:-1]] + [fine]
        ops = [capi.Operator.par(b2p_ctx, s.ndofs, s.ndofs, [coarsen(s)]) for s in spaces[:-1]]
        P = [common.gpu_interp(b2p_ctx, a, b, comps(x, y)) for a, b, x, y in zip(spaces[:-1], spaces[1:], orders[:-1], orders[1:])]
        return ops, P

    rt_ops, rt_P = levels(rt, lambda q: hs.build_rt_space(mesh, topo, q),
                          lambda s: rop.coarsen(s.p, s.ndofs, s.lex_gid, s.lex_sign, None, hs.tables_1d(s.p, q1d).Bo, hs.tables_1d(s.p, q1d).Bc,
                                                None), asm.rt_prolongation_comps)

    def nd_coarse(s):
        idx, ori = s.native_restriction()
        tt = hs.tables_1d(s.p, q1d)
        return mop.coarsen(s.p, s.ndofs, idx, ori, s.dof_map, tt.Bo, tt.Bc, tt.Gc)

    nd_ops, nd_P = levels(nd, lambda q: hs.build_nd_space(mesh, topo, q), nd_coarse, asm.nd_prolongation_comps)
    grad_est.set_multigrid(rt_ops + [Mrt], rt_P, coarse_type=1, coarse_tol=1e-8, coarse_max_it=2000)
    curl_est.set_multigrid(nd_ops + [Mnd], nd_P, coarse_type=1, coarse_tol=1e-8, coarse_max_it=2000)
    acc = np.zeros(ne)
    yr = torch.empty(rt.ndofs, dtype=torch.float64, device="cuda")
    mv = torch.empty(nd.ndofs, dtype=torch.float64, device="cuda")
    for v, lam in zip(c["modes"], c["lam"]):
        B = curl_dofs(nd, rt, v) / np.sqrt(lam / eps)
        Mnd.mult(_dev(v), mv)
        Mrt.mult(_dev(B), yr)
        Et = 0.5 * eps * float(v @ mv.cpu().numpy()) + 0.5 * float(B @ yr.cpu().numpy())
        D = torch.zeros(rt.ndofs, dtype=torch.float64, device="cuda")
        H = torch.zeros(nd.ndofs, dtype=torch.float64, device="cuda")
        est = torch.zeros(ne, dtype=torch.float64, device="cuda")
        grad_est.project(_dev(v), D)
        grad_est.integrate(_dev(v), D, est)
        curl_est.project(_dev(B), H)
        curl_est.integrate(_dev(B), H, est)
        assert grad_est.stats()["converged"] and curl_est.stats()["converged"]
        capi.flux_sqrt_scale(b2p_ctx, ne, 0.5 / Et, est)
        acc += est.cpu().numpy() ** 2
    e = np.sqrt(acc / len(c["modes"]))
    e_ref = oracle_indicators(c)
    assert np.abs(e - e_ref).max() < 1e-7 * e_ref.max()
    print("device indicator norm (tensor estimators, multigrid):", np.linalg.norm(e))
    if p == int(FIX["order"]):
        assert abs(np.linalg.norm(e) / REF_NORM - 1) < 1e-6


def test_refusals(b2p_ctx):
    from palace_b200 import capi

    c = case(b2p_ctx, 2, 3)
    I9 = np.eye(3).ravel()[None].repeat(3, axis=0)

    def refused(flux, smooth, code, words, M=None, geom=None):
        with pytest.raises(capi.B2PError) as ei:
            capi.FluxEstimator.hex(b2p_ctx, geom or c.geom, flux, smooth, I9, I9, I9, M or c.M["nd"])
        msg = str(ei.value)
        assert f"b2p error {code}:" in msg and all(w in msg for w in words), msg

    nd, rt = c.hex["nd"], c.hex["rt"]
    refused(rt, dict(nd, kind=capi.CURLCURL), 1, ["smooth space has kind 0", "B2P_ND_MASS"])
    refused(nd, nd, 1, ["both spaces are Nedelec"])
    refused(rt, dict(nd, p=3), 1, ["p=2", "p=3", "same"])
    refused(rt, dict(nd, idx=nd["idx"][:-1]), 1, ["smooth space has 8 elements vs 9 in the geometry"])
    refused(rt, nd, 1, ["no tensor q-data"], geom=capi.Geom.general(b2p_ctx, c.prob.qdata_ref))
    refused(rt, nd, 1, ["mass operator of the smooth space has the wrong size"], M=c.M["rt"])
    bad = np.array(nd["idx"], copy=True)
    bad[4, 5] = nd["lsize"]
    refused(rt, dict(nd, idx=bad), 1, ["smooth space", "outside L-vector"])
    refused(rt, dict(nd, assemble=True), 3, ["assembled q-data"])
    t3 = hs.tables_1d(2, 4)  # the tables of another quadrature, cut to this one's size
    refused(rt, dict(nd, Bo=t3.Bo[:3], Bc=t3.Bc[:3]), 1, ["Bo / Bc tables differ", "same 1-D tables"])
    # the kind is checked before anything the description asks for: a wrong kind with an unsupported order is still an argument error
    refused(dict(rt, kind=capi.CURLCURL, p=7), dict(nd, p=7), 1, ["flux space has kind 0"])

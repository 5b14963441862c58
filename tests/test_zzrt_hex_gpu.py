"""GPU: the sum-factorised Raviart-Thomas mass on hexahedra (kind B2P_RT_MASS, b2p_hex_flux.cu) against the oracle's H(div) mass matrix
and the dense-table operator, its diagonal, masked restriction, assembled RT_0 matrix, p-coarsening, refusals, and the grad-flux
estimator of the cylinder cavity with the sum-factorised RT mass under Jacobi and under the RT / ND p-multigrid. Bound: the operator
bound ||dy|| <= 1e-12 ||y|| unless stated otherwise."""
import os

import numpy as np
import pytest

from oracle import estimator as E
from palace_b200.host import assemble as asm
from palace_b200.host import coeff as cf
from palace_b200.host import hexmesh as hm
from palace_b200.host import hexspace as hs
from tests import common
from tests.test_cylinder_golden import FIX
from tests.test_cylinder_indicator_golden import REF_NORM, cavity_modes, curl_dofs, oracle_indicators

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

# anisotropic symmetric positive definite material tensors, one per attribute
_G = np.random.default_rng(7).standard_normal((3, 3, 3))
MATS = np.einsum("kij,klj->kil", _G, _G) + 2.0 * np.eye(3)[None]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return np.linalg.norm(a - b) / np.linalg.norm(b)


class Case:
    def __init__(self, ctx, p, q1d, n=(3, 2, 2), scramble=3):
        mesh = hm.box_mesh(n, (1.0, 0.7, 0.9), warp_amp=0.04, scramble_seed=scramble, n_attr=3)
        self.prob = common.problem_on_mesh(mesh, p=p, q1d=q1d)
        self.rt = hs.build_rt_space(mesh, self.prob.topo, p)
        self.p, self.q1d, self.ctx = p, q1d, ctx
        self.geom = common.gpu_geom(ctx, self.prob)
        self.blob = cf.coeff_ctx(np.arange(3), MATS)
        self.coef_elem = MATS[mesh.attr - 1]

    def op(self, p=None, assemble=False):
        from palace_b200 import capi

        rt = self.rt if p is None else hs.build_rt_space(self.prob.mesh, self.prob.topo, p)
        p = self.p if p is None else p
        t = hs.tables_1d(p, self.q1d)
        return capi.Op.create(self.ctx, self.geom, capi.RT_MASS, p, rt.ndofs, rt.lex_gid, rt.lex_sign, None, t.Bo, t.Bc, None, self.blob,
                              assemble)

    def oracle(self, sp=None):
        sp = self.rt if sp is None else sp
        B = E.rt_hex_tables(sp.p, self.q1d)
        s = sp.lex_sign.astype(float)
        return E.mixed_mass_matrix(self.prob.qdata_ref, B, E.HDIV, sp.lex_gid, s, sp.ndofs, B, E.HDIV, sp.lex_gid, s, sp.ndofs, self.coef_elem)

    def apply(self, op, x, **flags):
        y = torch.zeros(op.lsize, dtype=torch.float64, device="cuda")
        op.apply_add_ex(1.0, _dev(x), y, **flags)
        return y.cpu().numpy()


PQ = [(p, q) for p in range(1, 7) for q in (p + 1, p + 2) if q <= 7]


@pytest.mark.parametrize("p,q1d", PQ)
def test_parity_with_the_oracle_and_the_dense_operator(b2p_ctx, p, q1d):
    from palace_b200 import capi

    c = Case(b2p_ctx, p, q1d)
    op = c.op()
    x = np.random.default_rng(p + 10 * q1d).standard_normal(c.rt.ndofs)
    y = c.apply(op, x)
    y_ref = c.oracle() @ x
    assert _rel(y, y_ref) < 1e-12
    sp = dict(P=c.rt.P, map_type=capi.MAP_HDIV, interp=hs.rt_hex_dense_interp(p, q1d), idx=c.rt.lex_gid, orient=c.rt.lex_sign,
              lsize=c.rt.ndofs)
    Md = capi.vecfe_mass_operator(b2p_ctx, c.geom, sp, coef=np.stack([m.ravel(order="F") for m in MATS]))
    yd = torch.zeros(c.rt.ndofs, dtype=torch.float64, device="cuda")
    Md.mult(_dev(x), yd)
    assert _rel(y, yd.cpu().numpy()) < 1e-12


@pytest.mark.parametrize("p", [2, 3, 4, 5, 6])
def test_production_kernel_matches_the_cross_check_kernel(b2p_ctx, p):
    # 7 elements: a ragged last batch for every batch size of the production kernel (8, 4, 2, 2, 1 elements)
    c = Case(b2p_ctx, p, p + 1, n=(7, 1, 1), scramble=5)
    op = c.op()
    x = np.random.default_rng(p).standard_normal(c.rt.ndofs)
    y7, y1 = c.apply(op, x), c.apply(op, x, simple_kernel=True)
    assert _rel(y7, y1) < 1e-13
    assert _rel(y7, c.oracle() @ x) < 1e-12


@pytest.mark.parametrize("p", [1, 2, 4])
def test_diagonal(b2p_ctx, p):
    c = Case(b2p_ctx, p, p + 1)
    op = c.op()
    d = torch.zeros(c.rt.ndofs, dtype=torch.float64, device="cuda")
    op.diag_add(d)
    dr = c.oracle().diagonal()
    assert _rel(d.cpu().numpy(), dr) < 1e-12


@pytest.mark.parametrize("p", [1, 3])
@pytest.mark.parametrize("diag_policy", [1, 0])
def test_essential_face_dofs_match_the_eliminated_oracle(b2p_ctx, p, diag_policy):
    from palace_b200 import capi

    c = Case(b2p_ctx, p, p + 1)
    ess = c.rt.ess_dofs
    assert ess.size > 0
    A = capi.Operator.par(b2p_ctx, c.rt.ndofs, c.rt.ndofs, [c.op()], None, ess, diag_policy=diag_policy)
    x = np.random.default_rng(p).standard_normal(c.rt.ndofs)
    y = torch.zeros(c.rt.ndofs, dtype=torch.float64, device="cuda")
    A.mult(_dev(x), y)
    M = c.oracle().tolil()
    M[ess, :] = 0.0
    M[:, ess] = 0.0
    for i in ess:
        M[i, i] = float(diag_policy)
    assert _rel(y.cpu().numpy(), M.tocsr() @ x) < 1e-12


def test_rt0_assembled_matrix(b2p_ctx):
    from palace_b200 import capi

    c = Case(b2p_ctx, 1, 2)
    op = c.op()
    A = capi.Csr(b2p_ctx, op)
    A.assemble([op])
    Ad, Ar = A.to_scipy(), c.oracle()
    assert abs(Ad - Ar).max() < 1e-12 * abs(Ar).max()


@pytest.mark.parametrize("pc,pf", [(1, 2), (2, 4), (1, 4)])
def test_coarsened_operator_is_the_galerkin_product(b2p_ctx, pc, pf):
    from palace_b200 import capi

    c = Case(b2p_ctx, pf, pf + 1)
    fine = c.op()
    rc = hs.build_rt_space(c.prob.mesh, c.prob.topo, pc)
    t = hs.tables_1d(pc, c.q1d)
    coarse = fine.coarsen(pc, rc.ndofs, rc.lex_gid, rc.lex_sign, None, t.Bo, t.Bc, None)
    P = common.gpu_interp(b2p_ctx, rc, c.rt, asm.rt_prolongation_comps(pc, pf))
    x = np.random.default_rng(pc + pf).standard_normal(rc.ndofs)
    xf = torch.zeros(c.rt.ndofs, dtype=torch.float64, device="cuda")
    P.mult(_dev(x), xf)
    yf = torch.zeros_like(xf)
    fine.apply_add_ex(1.0, xf, yf)
    z = torch.zeros(rc.ndofs, dtype=torch.float64, device="cuda")
    P.mult_transpose(yf, z)
    yc = c.apply(coarse, x)
    assert _rel(z.cpu().numpy(), yc) < 1e-12
    assert _rel(yc, c.oracle(rc) @ x) < 1e-12


def test_refusals(b2p_ctx):
    from palace_b200 import capi

    c = Case(b2p_ctx, 2, 3)
    op = c.op()

    def refused(fn, code, words):
        with pytest.raises(capi.B2PError) as ei:
            fn()
        msg = str(ei.value)
        assert f"b2p error {code}:" in msg and all(w in msg for w in words), msg

    refused(lambda: c.op(assemble=True), 3, ["assembled q-data", "Raviart-Thomas"])
    refused(lambda: capi.Op.create_sum(b2p_ctx, [op, op], [1.0, 2.0]), 3, ["b2p_op_create_sum", "term 0"])
    n = c.rt.ndofs
    refused(lambda: capi.ComplexOperator.par(b2p_ctx, n, n, [op], [1.0 + 0.5j]), 3, ["b2p_coperator_par", "Raviart-Thomas"])
    x, y = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda")
    xg, yg = torch.zeros(4, dtype=torch.float64, device="cuda"), torch.zeros(4, dtype=torch.float64, device="cuda")
    refused(lambda: op.apply_add_split(1.0, x, xg, y, yg, n - 4, 0, c.prob.mesh.ne), 3, ["ghost pieces"])
    refused(lambda: capi.Op.create_dense(b2p_ctx, c.geom, capi.RT_MASS, n, c.rt.lex_gid, c.rt.lex_sign, hs.rt_hex_dense_interp(2, 3), None,
                                         c.blob), 1, ["bad kind"])
    # the multigrid of a flux estimator must end on the estimator's own smooth-space mass operator
    nd = c.prob.nd
    Mrt = capi.Operator.par(b2p_ctx, n, n, [op])
    other = capi.Operator.par(b2p_ctx, n, n, [c.op()])
    sp_rt = dict(P=c.rt.P, map_type=capi.MAP_HDIV, interp=hs.rt_hex_dense_interp(2, 3), idx=c.rt.lex_gid, orient=c.rt.lex_sign, lsize=n)
    sp_nd = dict(P=nd.P, map_type=capi.MAP_HCURL, interp=hs.nd_hex_dense_interp(2, 3), idx=nd.lex_gid, orient=nd.lex_sign, lsize=nd.ndofs)
    I9 = np.eye(3).ravel()[None].repeat(3, axis=0)
    est = capi.FluxEstimator(b2p_ctx, c.geom, sp_nd, sp_rt, I9, I9, I9, Mrt)
    refused(lambda: est.set_multigrid([other], []), 1, ["finest level"])


def _levels(ctx, fine_op, fine_space, orders, build_space, coarsen, comps):
    """Operators (coarse -> fine) and prolongations of a p-hierarchy that shares the fine operator's quadrature."""
    from palace_b200 import capi

    spaces = [build_space(q) for q in orders[:-1]] + [fine_space]
    ops = [capi.Operator.par(ctx, s.ndofs, s.ndofs, [coarsen(s)]) for s in spaces[:-1]]
    P = [common.gpu_interp(ctx, a, b, comps(x, y)) for a, b, x, y in zip(spaces[:-1], spaces[1:], orders[:-1], orders[1:])]
    return ops, P


def test_cylinder_grad_flux_estimator_with_the_sum_factorised_rt_mass(b2p_ctx):
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
    sp_rt = dict(P=rt.P, map_type=capi.MAP_HDIV, interp=hs.rt_hex_dense_interp(p, q1d), idx=rt.lex_gid, orient=rt.lex_sign, lsize=rt.ndofs)
    sp_nd = dict(P=nd.P, map_type=capi.MAP_HCURL, interp=hs.nd_hex_dense_interp(p, q1d), idx=nd.lex_gid, orient=nd.lex_sign, lsize=nd.ndofs)
    I9 = np.eye(3).ravel()[None]

    def estimators():
        curl_est = capi.FluxEstimator(b2p_ctx, geom, sp_rt, sp_nd, I9, I9, I9, Mnd, tol=1e-12, max_it=20000)
        grad_est = capi.FluxEstimator(b2p_ctx, geom, sp_nd, sp_rt, eps * I9, np.sqrt(eps) * I9, I9 / np.sqrt(eps), Mrt, tol=1e-12, max_it=20000)
        return grad_est, curl_est

    def indicators(grad_est, curl_est):
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
        return np.sqrt(acc / len(c["modes"])), grad_est.stats()["num_mult_its"]

    e_ref = oracle_indicators(c)
    # (a) the sum-factorised RT mass under Jacobi PCG
    e_jac, its_jac = indicators(*estimators())
    assert np.abs(e_jac - e_ref).max() < 1e-7 * e_ref.max()
    # (b) the same with the p-multigrid: RT levels for the grad-flux projection, ND levels for the curl-flux projection
    orders = asm.p_sequence(p)
    grad_est, curl_est = estimators()
    rt_ops, rt_P = _levels(b2p_ctx, rop, rt, orders, lambda q: hs.build_rt_space(mesh, topo, q),
                           lambda s: rop.coarsen(s.p, s.ndofs, s.lex_gid, s.lex_sign, None, hs.tables_1d(s.p, q1d).Bo,
                                                 hs.tables_1d(s.p, q1d).Bc, None), asm.rt_prolongation_comps)

    def nd_coarse(s):
        idx, ori = s.native_restriction()
        tt = hs.tables_1d(s.p, q1d)
        return mop.coarsen(s.p, s.ndofs, idx, ori, s.dof_map, tt.Bo, tt.Bc, tt.Gc)

    nd_ops, nd_P = _levels(b2p_ctx, mop, nd, orders, lambda q: hs.build_nd_space(mesh, topo, q), nd_coarse, asm.nd_prolongation_comps)
    grad_est.set_multigrid(rt_ops + [Mrt], rt_P, coarse_type=1, coarse_tol=1e-8, coarse_max_it=2000)
    curl_est.set_multigrid(nd_ops + [Mnd], nd_P, coarse_type=1, coarse_tol=1e-8, coarse_max_it=2000)
    e_mg, its_mg = indicators(grad_est, curl_est)
    assert np.abs(e_mg - e_ref).max() < 1e-7 * e_ref.max()
    print(f"grad-flux projection, {len(c['modes'])} modes, levels {orders}: Jacobi PCG {its_jac} iterations, multigrid PCG {its_mg}")
    print("device indicator norm (multigrid):", np.linalg.norm(e_mg))
    if p == int(FIX["order"]):
        assert abs(np.linalg.norm(e_mg) / REF_NORM - 1) < 1e-6
    # (c) the multigrid preconditioner pays for itself in iterations
    assert its_mg < its_jac

"""GPU: the sum-factorised discrete curl ND_p -> RT_{p-1} on hexahedra (b2p_interp_create_curl_hex, b2p_interp.cu). Mult and
MultTranspose against the assembled SciPy matrix of hexspace.discrete_curl_matrix with the reference's 1/multiplicity scaling, the
same curl as two Kronecker handles and as the element-dense interpolator, curl grad = 0, commuting with the ND / RT
p-prolongations, the true-dof operator wrapper, grids of several waves, the refusals, and B = curl E of the cylinder cavity fed to
the tensor flux estimators. Meshes are warped, with scrambled element frames, so shared faces and edges are seen with differing
local orientations. Bound: ||dy|| <= 1e-12 ||y|| unless stated otherwise."""
import ctypes as C

import numpy as np
import pytest

from oracle import solvers as S
from palace_b200.host import assemble as asm
from palace_b200.host import coeff as cf
from palace_b200.host import hexmesh as hm
from palace_b200.host import hexspace as hs
from tests import common
from tests.test_cylinder_golden import FIX
from tests.test_cylinder_indicator_golden import REF_NORM, cavity_modes, curl_dofs, oracle_indicators

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ALPHA = -0.7


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return np.linalg.norm(a - b) / np.linalg.norm(b)


class Mesh:
    """ND_p and RT_{p-1} (and H1_p on request) on one warped, scrambled box mesh."""

    def __init__(self, p, n=(3, 2, 2), scramble=3):
        self.p = p
        self.mesh = hm.box_mesh(n, (1.0, 0.7, 0.9), warp_amp=0.04, scramble_seed=scramble, n_attr=3)
        self.topo = hs.build_topology(self.mesh)
        self.nd = hs.build_nd_space(self.mesh, self.topo, p)
        self.rt = hs.build_rt_space(self.mesh, self.topo, p)

    def curl(self, ctx):
        from palace_b200 import capi

        return capi.Interp.curl_hex(ctx, asm.space_dict(self.nd), asm.space_dict(self.rt), self.p)

    def kron(self, ctx):
        """The same curl as two b2p_interp_create handles, one per term."""
        from palace_b200 import capi

        return [capi.Interp(ctx, asm.space_dict(self.nd), asm.space_dict(self.rt), t) for t in asm.curl_kron_terms(self.p)]

    def dense(self, ctx):
        from palace_b200 import capi

        nd, rt = self.nd, self.rt
        return capi.Interp.dense(ctx, hs.discrete_curl_matrix(self.p), nd.lex_gid, nd.ndofs, rt.lex_gid, rt.ndofs, in_orient=nd.lex_sign,
                                 out_orient=rt.lex_sign)

    def matrix(self):
        """(1/mult_rt) sum_e E_rt^T C_e E_nd as a SciPy matrix."""
        nd, rt = self.nd, self.rt
        return S.interp_matrix(hs.discrete_curl_matrix(self.p), nd.lex_gid, nd.lex_sign.astype(float), rt.lex_gid, rt.lex_sign.astype(float),
                               nd.ndofs, rt.ndofs)

    def element_apply(self, x, transpose):
        """The same products element by element (no global matrix): for meshes too large for the SciPy matrix."""
        nd, rt, Cl = self.nd, self.rt, hs.discrete_curl_matrix(self.p)
        inv = 1.0 / np.bincount(rt.lex_gid.ravel(), minlength=rt.ndofs)
        if not transpose:
            ye = (nd.lex_sign * x[nd.lex_gid]) @ Cl.T * rt.lex_sign
            return inv * np.bincount(rt.lex_gid.ravel(), weights=ye.ravel(), minlength=rt.ndofs)
        ye = (rt.lex_sign * (inv * x)[rt.lex_gid]) @ Cl * nd.lex_sign
        return np.bincount(nd.lex_gid.ravel(), weights=ye.ravel(), minlength=nd.ndofs)

    def sizes(self, transpose):
        return (self.rt.ndofs, self.nd.ndofs) if transpose else (self.nd.ndofs, self.rt.ndofs)


def apply(its, x, y0, transpose=False, alpha=ALPHA):
    y = _dev(y0)
    for it in its:
        it.apply_add(_dev(x), y, transpose=transpose, alpha=alpha)
    return y.cpu().numpy()


_meshes = {}


def mesh(p):
    if p not in _meshes:
        _meshes[p] = Mesh(p)
    return _meshes[p]


@pytest.mark.parametrize("p", range(1, 7))
@pytest.mark.parametrize("transpose", [False, True])
def test_apply_matches_the_assembled_curl(b2p_ctx, p, transpose):
    m = mesh(p)
    n_in, n_out = m.sizes(transpose)
    rng = np.random.default_rng(10 * p + transpose)
    x, y0 = rng.standard_normal(n_in), rng.standard_normal(n_out)
    y = apply([m.curl(b2p_ctx)], x, y0, transpose)
    Cm = m.matrix()
    # MultTranspose scales its input by 1/mult_rt: (diag(1/mult) M)^T x = M^T ((1/mult) x)
    y_ref = y0 + ALPHA * ((Cm.T @ x) if transpose else (Cm @ x))
    assert _rel(y - y0, y_ref - y0) < 1e-12
    assert _rel(y, y_ref) < 1e-12


@pytest.mark.parametrize("p", range(1, 7))
def test_agrees_with_the_two_handle_and_dense_routes(b2p_ctx, p):
    m = mesh(p)
    curl, kron = m.curl(b2p_ctx), m.kron(b2p_ctx)
    dense = m.dense(b2p_ctx) if p <= 4 else None
    for transpose in (False, True):
        n_in, n_out = m.sizes(transpose)
        rng = np.random.default_rng(p + 20 * transpose)
        x, y0 = rng.standard_normal(n_in), rng.standard_normal(n_out)
        y = apply([curl], x, y0, transpose) - y0
        assert _rel(y, apply(kron, x, y0, transpose) - y0) < 1e-14
        if dense is not None:
            assert _rel(y, apply([dense], x, y0, transpose) - y0) < 1e-14


def test_dense_route_refuses_the_orders_the_curl_kernel_covers(b2p_ctx):
    from palace_b200 import capi

    with pytest.raises(capi.B2PError, match="element too large"):
        mesh(5).dense(b2p_ctx)


@pytest.mark.parametrize("p", range(1, 7))
def test_curl_of_a_gradient_vanishes(b2p_ctx, p):
    from palace_b200 import capi

    m = mesh(p)
    h1 = hs.build_h1_space(m.mesh, m.topo, p)
    G = capi.Interp(b2p_ctx, asm.space_dict(h1), asm.space_dict(m.nd), asm.gradient_comps(p))
    phi = _dev(np.random.default_rng(p).standard_normal(h1.ndofs))
    g = torch.zeros(m.nd.ndofs, dtype=torch.float64, device="cuda")
    G.apply_add(phi, g)
    b = torch.zeros(m.rt.ndofs, dtype=torch.float64, device="cuda")
    m.curl(b2p_ctx).apply_add(g, b)
    assert np.linalg.norm(b.cpu().numpy()) <= 1e-12 * np.linalg.norm(g.cpu().numpy())


PAIRS = sorted({pr for q in (6, 4) for pr in zip(asm.p_sequence(q)[:-1], asm.p_sequence(q)[1:])})


@pytest.mark.parametrize("pc,pf", PAIRS)
def test_curl_commutes_with_the_p_prolongations(b2p_ctx, pc, pf):
    from palace_b200 import capi

    mf = mesh(pf)
    nd_c, rt_c = hs.build_nd_space(mf.mesh, mf.topo, pc), hs.build_rt_space(mf.mesh, mf.topo, pc)
    Pnd = capi.Interp(b2p_ctx, asm.space_dict(nd_c), asm.space_dict(mf.nd), asm.nd_prolongation_comps(pc, pf))
    Prt = capi.Interp(b2p_ctx, asm.space_dict(rt_c), asm.space_dict(mf.rt), asm.rt_prolongation_comps(pc, pf))
    Cc = capi.Interp.curl_hex(b2p_ctx, asm.space_dict(nd_c), asm.space_dict(rt_c), pc)
    x = _dev(np.random.default_rng(pc + 10 * pf).standard_normal(nd_c.ndofs))
    xf = torch.zeros(mf.nd.ndofs, dtype=torch.float64, device="cuda")
    Pnd.apply_add(x, xf)
    lhs = torch.zeros(mf.rt.ndofs, dtype=torch.float64, device="cuda")
    mf.curl(b2p_ctx).apply_add(xf, lhs)
    bc = torch.zeros(rt_c.ndofs, dtype=torch.float64, device="cuda")
    Cc.apply_add(x, bc)
    rhs = torch.zeros(mf.rt.ndofs, dtype=torch.float64, device="cuda")
    Prt.apply_add(bc, rhs)
    assert _rel(lhs.cpu().numpy(), rhs.cpu().numpy()) < 1e-12


@pytest.mark.parametrize("p", [2, 5])
def test_true_dof_operator_equals_the_raw_apply(b2p_ctx, p):
    from palace_b200 import capi

    m = mesh(p)
    it = m.curl(b2p_ctx)
    op = capi.Operator.interp(b2p_ctx, it)
    rng = np.random.default_rng(p)
    for transpose in (False, True):
        n_in, n_out = m.sizes(transpose)
        x = rng.standard_normal(n_in)
        y = torch.full((n_out,), np.nan, dtype=torch.float64, device="cuda")  # overwritten, not accumulated
        (op.mult_transpose if transpose else op.mult)(_dev(x), y)
        y_raw = apply([it], x, np.zeros(n_out), transpose, alpha=1.0)
        assert np.array_equal(y.cpu().numpy(), y_raw) or _rel(y.cpu().numpy(), y_raw) < 1e-15


@pytest.mark.parametrize("p,n", [(3, (23, 23, 23)), (6, (13, 13, 13))])
def test_grids_of_several_waves(b2p_ctx, p, n):
    # p = 3: 12167 elements, 5 (Mult) and 4 (MultTranspose) elements per block, so the last block is partly filled; p = 6: one
    # element per block. Both give more blocks than an H100 holds at once.
    m = Mesh(p, n=n, scramble=7)
    curl, kron = m.curl(b2p_ctx), m.kron(b2p_ctx)
    for transpose in (False, True):
        n_in, n_out = m.sizes(transpose)
        rng = np.random.default_rng(p + transpose)
        x, y0 = rng.standard_normal(n_in), rng.standard_normal(n_out)
        y = apply([curl], x, y0, transpose)
        assert _rel(y - y0, ALPHA * m.element_apply(x, transpose)) < 1e-12
        assert _rel(y - y0, apply(kron, x, y0, transpose) - y0) < 1e-14


def test_refusals(b2p_ctx):
    from palace_b200 import capi

    m = mesh(2)
    p, nd, rt = 2, asm.space_dict(m.nd), asm.space_dict(m.rt)
    keep = []
    dtypes = dict(nd_idx=np.int32, nd_orient=np.int8, nd_dof_map=np.int32, rt_idx=np.int32, rt_orient=np.int8, rt_dof_map=np.int32,
                  D=np.float64)

    def desc(**over):
        d = capi.CurlInterpDesc()
        f = dict(ne=m.mesh.ne, p=p, nd_lsize=nd["lsize"], nd_idx=nd["idx"], nd_orient=nd["orient"], nd_dof_map=nd["dof_map"],
                 rt_lsize=rt["lsize"], rt_idx=rt["idx"], rt_orient=rt["orient"], rt_dof_map=None, D=asm.curl_table(p))
        f.update(over)
        for k, v in f.items():
            if isinstance(v, np.ndarray):
                v = np.ascontiguousarray(v, dtype=dtypes[k])
                keep.append(v)
                v = v.ctypes.data
            setattr(d, k, v)
        return d

    def refused(d, code, words, ctx=b2p_ctx):
        h = C.c_void_p()
        rc = capi.lib().b2p_interp_create_curl_hex(ctx.h if ctx else None, C.byref(d) if d is not None else None, C.byref(h))
        msg = capi.lib().b2p_last_error(ctx.h if ctx else None).decode()
        assert rc == code and all(w in msg for w in words), (rc, msg)
        assert not h.value

    refused(None, 1, ["b2p_interp_create_curl_hex", "null argument"])
    refused(desc(), 1, ["null argument"], ctx=None)
    for field in ("nd_idx", "rt_idx", "D"):
        refused(desc(**{field: None}), 1, ["null argument"])
    refused(desc(ne=0), 1, ["no elements"])
    refused(desc(p=0), 1, ["p=0", "at least 1"])
    refused(desc(p=7), 3, ["p=7", "1..6"])
    refused(desc(rt_lsize=0), 1, ["rt_lsize=0"])
    bad = np.array(nd["idx"], copy=True)
    bad[3, 5] = nd["lsize"]
    refused(desc(nd_idx=bad), 1, ["idx out of range"])
    bad = np.array(rt["idx"], copy=True)
    bad[2, 1] = -1
    refused(desc(rt_idx=bad), 1, ["idx out of range"])  # after the ND restriction is on the device: it is freed
    bad = np.array(nd["dof_map"], copy=True)
    bad[4] = m.nd.P
    refused(desc(nd_dof_map=bad), 1, ["dof_map[4] out of range"])
    bad = np.zeros(m.rt.P, dtype=np.int32)
    bad[0] = -1 - m.rt.P
    refused(desc(rt_dof_map=bad), 1, ["dof_map[0] out of range"])
    # the Python layer checks the shapes the C ABI cannot see
    with pytest.raises(ValueError, match="rt idx has shape"):
        capi.Interp.curl_hex(b2p_ctx, nd, dict(rt, idx=rt["idx"][:, :-1]), p)
    # a valid description still builds after the refusals
    h = C.c_void_p()
    assert capi.lib().b2p_interp_create_curl_hex(b2p_ctx.h, C.byref(desc()), C.byref(h)) == 0
    capi.lib().b2p_interp_destroy(h)


def test_cylinder_estimators_fed_by_the_device_curl(b2p_ctx):
    """B = curl E / sqrt(lam / eps) of the cylinder cavity's modes at order 4 from the device curl, fed unchanged to the tensor flux
    estimators with the RT / ND p-multigrid projections: the indicators and the reference's global norm as with the host curl."""
    from palace_b200 import capi

    p = int(FIX["order"])
    c = cavity_modes(p)
    mesh_, topo, nd, rt, q1d, eps = c["mesh"], c["topo"], c["nd"], c["rt"], c["q1d"], c["eps"]
    ne = mesh_.ne
    curl = capi.Interp.curl_hex(b2p_ctx, asm.space_dict(nd), asm.space_dict(rt), p)
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

    rt_ops, rt_P = levels(rt, lambda q: hs.build_rt_space(mesh_, topo, q),
                          lambda s: rop.coarsen(s.p, s.ndofs, s.lex_gid, s.lex_sign, None, hs.tables_1d(s.p, q1d).Bo, hs.tables_1d(s.p, q1d).Bc,
                                                None), asm.rt_prolongation_comps)

    def nd_coarse(s):
        idx, ori = s.native_restriction()
        tt = hs.tables_1d(s.p, q1d)
        return mop.coarsen(s.p, s.ndofs, idx, ori, s.dof_map, tt.Bo, tt.Bc, tt.Gc)

    nd_ops, nd_P = levels(nd, lambda q: hs.build_nd_space(mesh_, topo, q), nd_coarse, asm.nd_prolongation_comps)
    grad_est.set_multigrid(rt_ops + [Mrt], rt_P, coarse_type=1, coarse_tol=1e-8, coarse_max_it=2000)
    curl_est.set_multigrid(nd_ops + [Mnd], nd_P, coarse_type=1, coarse_tol=1e-8, coarse_max_it=2000)
    acc = np.zeros(ne)
    yr = torch.empty(rt.ndofs, dtype=torch.float64, device="cuda")
    mv = torch.empty(nd.ndofs, dtype=torch.float64, device="cuda")
    for v, lam in zip(c["modes"], c["lam"]):
        E = _dev(v)
        B = torch.zeros(rt.ndofs, dtype=torch.float64, device="cuda")
        curl.apply_add(E, B, alpha=1.0 / np.sqrt(lam / eps))
        B_host = curl_dofs(nd, rt, v) / np.sqrt(lam / eps)
        assert _rel(B.cpu().numpy(), B_host) < 1e-13
        Mnd.mult(E, mv)
        Mrt.mult(B, yr)
        Et = 0.5 * eps * float(v @ mv.cpu().numpy()) + 0.5 * float(torch.dot(B, yr))
        D = torch.zeros(rt.ndofs, dtype=torch.float64, device="cuda")
        H = torch.zeros(nd.ndofs, dtype=torch.float64, device="cuda")
        est = torch.zeros(ne, dtype=torch.float64, device="cuda")
        grad_est.project(E, D)
        grad_est.integrate(E, D, est)
        curl_est.project(B, H)
        curl_est.integrate(B, H, est)
        assert grad_est.stats()["converged"] and curl_est.stats()["converged"]
        capi.flux_sqrt_scale(b2p_ctx, ne, 0.5 / Et, est)
        acc += est.cpu().numpy() ** 2
    e = np.sqrt(acc / len(c["modes"]))
    e_ref = oracle_indicators(c)
    assert np.abs(e - e_ref).max() < 1e-7 * e_ref.max()
    assert abs(np.linalg.norm(e) / REF_NORM - 1) < 1e-6

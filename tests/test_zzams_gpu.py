"""GPU: the algebraic coarse solvers (b2p_solver_amg / b2p_solver_ams) against their oracle (oracle/amg.py) and in the wirings
Palace uses them in: as the assembled coarse solver of the p-multigrid, through b2p_ksp_create's coarse_type 2, under
b2p_divfree and inside b2p_csolver_assembled.

The oracle builds its hierarchies from the very matrix the device holds (Csr.to_scipy), so the aggregation sees the same numbers
and the levels agree exactly; the solve phase agrees to round-off."""
import functools
import os

import numpy as np
import pytest
import scipy.sparse.linalg as spla

from oracle import amg
from oracle import pyoracle as O
from oracle import solvers as S
from palace_b200.host import assemble as asm
from palace_b200.host import hexspace as hs
from tests import common

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
EMU = os.environ.get("B2P_EMU_TESTS") == "1"


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _host(t):
    return t.cpu().numpy()


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def _gradient(prob, nd=None, h1=None):
    nd = prob.nd if nd is None else nd
    h1 = prob.h1 if h1 is None else h1
    return common.oracle_interp(h1, nd, hs.discrete_gradient_matrix(1))


@functools.lru_cache(maxsize=None)
def _box(n):
    return common.make_problem(n=(n, n, n), p=1, warp=0.04, scramble=3, n_attr=3)


def _device_matrix(ctx, prob, kind, blob, space):
    """Device-assembled, eliminated matrix (b2p_csr) and its operator."""
    from palace_b200 import capi

    geom = common.gpu_geom(ctx, prob)
    op = common.gpu_op(ctx, geom, prob, kind, blob, space=space)
    csr = capi.Csr(ctx, op)
    csr.assemble([op])
    csr.eliminate(space.ess_dofs, diag_policy=1)
    A = capi.Operator.from_csr(ctx, csr)
    A.keep = [geom, op, csr]
    return A, csr.to_scipy()


@pytest.fixture(scope="module")
def nd_box(b2p_ctx):
    prob = _box(8)
    A, Ah = _device_matrix(b2p_ctx, prob, O.CURLCURL_MASS, common.coefficient(O.CURLCURL_MASS, 3, "matrix"), prob.nd)
    return dict(prob=prob, A=A, Ah=Ah, G=_gradient(prob), X=amg.vertex_coords(prob.mesh))


@pytest.fixture(scope="module")
def h1_box(b2p_ctx):
    prob = _box(8)
    A, Ah = _device_matrix(b2p_ctx, prob, O.H1_DIFFUSION, common.coefficient(O.H1_DIFFUSION, 3, "matrix"), prob.h1)
    return dict(prob=prob, A=A, Ah=Ah)


def _ams(ctx, s, cycle_it=1, smooth_it=1, singular=False):
    from palace_b200 import capi

    dev = capi.Solver.ams(ctx, s["G"], s["X"], cycle_it=cycle_it, smooth_it=smooth_it, singular=singular)
    dev.set_operator(s["A"])
    return dev, amg.AMS(s["Ah"], s["G"], s["X"], cycle_it=cycle_it, smooth_it=smooth_it, singular=singular)


def _amg(ctx, s, cycle_it=1, smooth_it=1):
    from palace_b200 import capi

    dev = capi.Solver.amg(ctx, cycle_it=cycle_it, smooth_it=smooth_it)
    dev.set_operator(s["A"])
    return dev, amg.AMG(s["Ah"], cycle_it=cycle_it, smooth_it=smooth_it)


# ---------------------------------------------------------------------------------------------------- 1. hierarchies
def test_levels_equal_the_oracle(b2p_ctx, nd_box, h1_box):
    from palace_b200 import capi

    capi.set_stream(b2p_ctx)
    dev, ref = _amg(b2p_ctx, h1_box)
    assert dev.levels(0) == (ref.H.rows, ref.H.nnz)
    assert len(ref.H.rows) >= 2
    dev, ref = _ams(b2p_ctx, nd_box)
    for h, H in enumerate(ref.hierarchies()):
        assert dev.levels(h) == (H.rows, H.nnz), h
        assert len(H.rows) >= 2
    print("AMS hierarchies (rows):", [H.rows for H in ref.hierarchies()], "setup", round(dev.setup_ms(), 1), "ms")
    sing, ref_s = _ams(b2p_ctx, nd_box, singular=True)
    assert sing.levels(0) == ([], [])
    assert sing.levels(1) == (ref_s.HPi[0].rows, ref_s.HPi[0].nnz)


# ---------------------------------------------------------------------------------------------------- 2. one Mult
@pytest.mark.parametrize("cycle_it,smooth_it", [(1, 1), (1, 2), (2, 1), (2, 2)])
@pytest.mark.parametrize("which", ["amg", "ams"])
def test_mult_equals_the_oracle(b2p_ctx, nd_box, h1_box, which, cycle_it, smooth_it):
    from palace_b200 import capi

    capi.set_stream(b2p_ctx)
    s = h1_box if which == "amg" else nd_box
    dev, ref = (_amg if which == "amg" else _ams)(b2p_ctx, s, cycle_it, smooth_it)
    n = s["Ah"].shape[0]
    b = np.random.default_rng(5).standard_normal(n)
    y = torch.full((n,), 7.0, dtype=torch.float64, device="cuda")  # overwritten: no initial guess
    dev.mult(_dev(b), y)
    first = _host(y)
    err = _rel(first, ref.mult(b))
    assert err < 1e-12, err
    dev.mult(_dev(b), y)
    assert np.array_equal(_host(y), first)
    # with the initial guess the cycles continue from y
    dev.set_initial_guess(1)
    x0 = np.random.default_rng(6).standard_normal(n)
    y.copy_(_dev(x0))
    dev.mult(_dev(b), y)
    assert _rel(_host(y), ref.mult(b, x0)) < 1e-12


# ---------------------------------------------------------------------------------------------------- 3. CG + AMS
def test_device_cg_with_ams_takes_the_oracle_iterations(b2p_ctx, nd_box):
    from palace_b200 import capi

    capi.set_stream(b2p_ctx)
    dev, ref = _ams(b2p_ctx, nd_box)
    n = nd_box["Ah"].shape[0]
    b = np.random.default_rng(7).standard_normal(n)
    b[nd_box["prob"].nd.ess_dofs] = 0.0
    cg = capi.Solver.krylov(b2p_ctx, capi.CG, rel_tol=1e-8, max_it=500)
    cg.set_operator(nd_box["A"])
    cg.set_preconditioner(dev)
    x = torch.zeros(n, dtype=torch.float64, device="cuda")
    cg.mult(_dev(b), x)
    st = cg.stats()
    _, it_ref, _ = S.cg(nd_box["Ah"], b, ref, rel_tol=1e-8, max_it=500)
    assert st["converged"] and abs(st["its"] - it_ref) <= 1, (st, it_ref)
    assert _rel(nd_box["Ah"] @ _host(x), b) < 1e-7


# ---------------------------------------------------------------------------------------------------- 5. b2p_ksp coarse_type 2
def test_ksp_coarse_type_2_with_assembled_ams(b2p_ctx):
    from palace_b200 import capi

    capi.set_stream(b2p_ctx)
    prob = _box(6)
    blob = common.coefficient(O.CURLCURL_MASS, 3, "matrix")
    geom = common.gpu_geom(b2p_ctx, prob)
    A = common.gpu_par_operator(b2p_ctx, geom, prob, O.CURLCURL_MASS, blob)
    ams = capi.Solver.ams(b2p_ctx, _gradient(prob), amg.vertex_coords(prob.mesh))
    coarse = capi.Solver.assembled(b2p_ctx, ams)
    ksp = capi.Ksp(b2p_ctx, 1, coarse_solver=coarse, krylov_solver=capi.CG, coarse_type=2, tol=1e-10, max_it=200)
    ksp.set_operators(A, [A])
    n = prob.nd.ndofs
    b = np.random.default_rng(8).standard_normal(n)
    b[prob.nd.ess_dofs] = 0.0
    x = torch.zeros(n, dtype=torch.float64, device="cuda")
    ksp.mult(_dev(b), x)
    st = ksp.stats()
    Ao = common.oracle_matrix(prob, O.CURLCURL_MASS, blob)
    assert st["converged"] and st["its"] < 40, st
    assert _rel(_host(x), spla.spsolve(Ao.tocsc(), b)) < 1e-8


# ---------------------------------------------------------------------------------------------------- 4. cylinder cavity
def test_cylinder_cavity_with_ams_coarse_solver(b2p_ctx):
    from palace_b200 import capi
    from palace_b200.host import coeff as cf
    from tests.test_cylinder_golden import FIX, frequencies_ghz, target_lambda
    from tests.test_zcylinder_gpu import _problem

    capi.set_stream(b2p_ctx)
    p, nev = int(FIX["order"]), 3
    prob = _problem(p)
    geom = common.gpu_geom(b2p_ctx, prob)
    orders = asm.p_sequence(p)
    nd = {q: (prob.nd if q == p else hs.build_nd_space(prob.mesh, prob.topo, q)) for q in orders}
    h1 = {q: (prob.h1 if q == p else hs.build_h1_space(prob.mesh, prob.topo, q)) for q in orders}
    sigma = target_lambda()
    ident = cf.coeff_ctx()
    blob_A = cf.coeff_ctx_pair(cf.coeff_ctx(a=-sigma), cf.coeff_ctx(a=1.0))
    blob_P = cf.coeff_ctx_pair(cf.coeff_ctx(a=+sigma), cf.coeff_ctx(a=1.0))
    blob_G = cf.coeff_ctx(a=sigma)
    M = common.gpu_par_operator(b2p_ctx, geom, prob, O.ND_MASS, ident, space=nd[p])
    A = common.gpu_par_operator(b2p_ctx, geom, prob, O.CURLCURL_MASS, blob_A, space=nd[p])
    Pl = {p: common.gpu_par_operator(b2p_ctx, geom, prob, O.CURLCURL_MASS, blob_P, space=nd[p])}
    AG = {p: common.gpu_par_operator(b2p_ctx, geom, prob, O.H1_DIFFUSION, blob_G, space=h1[p])}
    for q in orders[:-1]:
        Pl[q] = common.gpu_par_operator(b2p_ctx, geom, prob, O.CURLCURL_MASS, blob_P, space=nd[q], fine_op=Pl[p].local_op)
        AG[q] = common.gpu_par_operator(b2p_ctx, geom, prob, O.H1_DIFFUSION, blob_G, space=h1[q], fine_op=AG[p].local_op)
    G = [common.gpu_interp(b2p_ctx, h1[q], nd[q], asm.gradient_comps(q)) for q in orders]
    P = [common.gpu_interp(b2p_ctx, nd[a], nd[b], asm.nd_prolongation_comps(a, b)) for a, b in zip(orders[:-1], orders[1:])]
    # vertex coordinates: the corners of the second-order element nodes (lexicographic, 3 per direction)
    xe2 = np.asarray(FIX["xe2"])
    X = np.zeros((h1[1].ndofs, 3))
    for c in range(8):
        a, b_, cc = c & 1, (c >> 1) & 1, (c >> 2) & 1
        X[prob.mesh.elems[:, c]] = xe2[:, :, 2 * a + 3 * 2 * b_ + 9 * 2 * cc]
    ams = capi.Solver.ams(b2p_ctx, _gradient(prob, nd[1], h1[1]), X, cycle_it=p)
    coarse = capi.Solver.assembled(b2p_ctx, ams)
    mg = capi.Solver.gmg(b2p_ctx, coarse, P, G, cycle_it=2, smooth_it=1, cheby_order=6)
    mg.gmg_set_operators([Pl[q] for q in orders], [AG[q] for q in orders])
    ksp = capi.Solver.krylov(b2p_ctx, capi.FGMRES, rel_tol=1e-12, max_it=300, max_dim=300)
    ksp.set_operator(A)
    ksp.set_preconditioner(mg)
    n = nd[p].ndofs
    free = np.setdiff1d(np.arange(n), nd[p].ess_dofs)
    xd = torch.zeros(n, dtype=torch.float64, device="cuda")
    yd = torch.zeros(n, dtype=torch.float64, device="cuda")
    its = []

    def to_full(v):
        f = np.zeros(n)
        f[free] = v
        return f

    def opinv(v):
        xd.copy_(torch.from_numpy(to_full(v)))
        ksp.mult(xd, yd)
        its.append(ksp.stats()["its"])
        return yd.cpu().numpy()[free]

    def mmul(v):
        xd.copy_(torch.from_numpy(to_full(v)))
        M.mult(xd, yd)
        return yd.cpu().numpy()[free]

    nf = free.size
    Kop = spla.LinearOperator((nf, nf), matvec=lambda v: None, dtype=np.float64)
    lam = spla.eigsh(Kop, k=nev, M=spla.LinearOperator((nf, nf), matvec=mmul, dtype=np.float64), sigma=sigma, which="LA",
                     OPinv=spla.LinearOperator((nf, nf), matvec=opinv, dtype=np.float64), tol=1e-11,
                     v0=np.random.default_rng(0).standard_normal(nf), return_eigenvectors=False)
    f = frequencies_ghz(np.sort(lam))
    rel = np.abs(f.real - FIX["ref_f_re_ghz"][:nev]) / FIX["ref_f_re_ghz"][:nev]
    print("cylinder, AMS coarse solver: rel. error vs eig.csv", rel, " FGMRES its/solve:", np.mean(its), "AMS levels",
          [mg.levels(h)[0] for h in range(4)])
    assert rel.max() < 1e-8


# ---------------------------------------------------------------------------------------------------- 6. divfree
def test_divfree_with_amg_coarse_solver_matches_jacobi_pcg(b2p_ctx):
    from palace_b200 import capi

    capi.set_stream(b2p_ctx)
    prob = common.make_problem(n=(5, 4, 4), p=2)
    p = 2
    geom = common.gpu_geom(b2p_ctx, prob)
    blob = common.coefficient(O.ND_MASS, 3, "matrix", a_mass=1.3)
    orders = asm.p_sequence(p)
    h1 = {q: (prob.h1 if q == p else hs.build_h1_space(prob.mesh, prob.topo, q)) for q in orders}
    mop = common.gpu_op(b2p_ctx, geom, prob, O.ND_MASS, blob)
    Mnd = capi.Operator.par(b2p_ctx, prob.nd.ndofs, prob.nd.ndofs, [mop], None, None, diag_policy=1)
    G = common.gpu_interp(b2p_ctx, h1[p], prob.nd, asm.gradient_comps(p))
    fineK = common.gpu_par_operator(b2p_ctx, geom, prob, O.H1_DIFFUSION, blob, space=h1[p])
    K = [fineK if q == p else common.gpu_par_operator(b2p_ctx, geom, prob, O.H1_DIFFUSION, blob, space=h1[q], fine_op=fineK.local_op)
         for q in orders]
    P = [common.gpu_interp(b2p_ctx, h1[a], h1[b], asm.h1_prolongation_comps(a, b)) for a, b in zip(orders[:-1], orders[1:])]
    y = np.random.default_rng(9).standard_normal(prob.nd.ndofs)
    out = []
    for kind in ("jacobi_pcg", "amg"):
        kw = dict(coarse_type=1, coarse_tol=1e-3) if kind == "jacobi_pcg" else dict(
            coarse_type=2, coarse_solver=capi.Solver.assembled(b2p_ctx, capi.Solver.amg(b2p_ctx)))
        dv = capi.DivFree(b2p_ctx, Mnd, G, K, P, h1[p].ess_dofs, p, tol=1e-11, max_it=200, **kw)
        yd = _dev(y)
        dv.mult(yd)
        assert dv.stats()["converged"], kind
        out.append(_host(yd))
    assert _rel(out[1], out[0]) < 1e-9


# ---------------------------------------------------------------------------------------------------- 7. complex wrapper
def test_csolver_assembled_with_ams_on_a_lossy_shifted_operator(b2p_ctx):
    from palace_b200 import capi
    from tests.test_zzcomplex_assembled_gpu import _complex_op, _parts_ref, lossy_problem

    capi.set_stream(b2p_ctx)
    prob, terms, coefs = lossy_problem(1)
    A = _complex_op(b2p_ctx, prob, terms, coefs)
    ams = capi.Solver.ams(b2p_ctx, _gradient(prob), amg.vertex_coords(prob.mesh))
    pc = capi.ComplexSolver.assembled(b2p_ctx, ams)
    pc.set_operator(A)
    Ks = capi.ComplexSolver.krylov(b2p_ctx, capi.GMRES, rel_tol=1e-10, max_it=300, max_dim=300)
    Ks.set_operator(A)
    Ks.set_preconditioner(pc)
    n = prob.nd.ndofs
    rng = np.random.default_rng(10)
    b = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    b[prob.nd.ess_dofs] = 0.0
    zr, zi = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda")
    Ks.mult(_dev(b.real), _dev(b.imag), zr, zi)
    st = Ks.stats()
    Ar, Ai = _parts_ref(prob, terms, coefs)
    x = spla.spsolve((Ar + 1j * Ai).tocsc(), b)
    print("lossy cavity p = 1, GMRES + assembled Ar + Ai AMS:", st)
    assert st["converged"] and _rel(_host(zr) + 1j * _host(zi), x) < 1e-8, st


# ---------------------------------------------------------------------------------------------------- 8. error paths
def test_error_paths(b2p_ctx, nd_box):
    from palace_b200 import capi

    capi.set_stream(b2p_ctx)
    prob = nd_box["prob"]
    geom = common.gpu_geom(b2p_ctx, prob)
    par = common.gpu_par_operator(b2p_ctx, geom, prob, O.CURLCURL_MASS, common.coefficient(O.CURLCURL_MASS, 3, "matrix"))
    n = prob.nd.ndofs
    x, y = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda")
    for s in (capi.Solver.amg(b2p_ctx), capi.Solver.ams(b2p_ctx, nd_box["G"], nd_box["X"])):
        with pytest.raises(capi.B2PError, match="before SetOperator"):
            s.mult(x, y)
        with pytest.raises(capi.B2PError, match="assembled real matrix"):
            s.set_operator(par)
        with pytest.raises(capi.B2PError, match="before SetOperator"):
            s.mult(x, y)
    small = _box(4)
    bad = capi.Solver.ams(b2p_ctx, _gradient(small), amg.vertex_coords(small.mesh))
    with pytest.raises(capi.B2PError, match="discrete gradient"):
        bad.set_operator(nd_box["A"])
    Gs = nd_box["G"].tocsr()
    with pytest.raises(capi.B2PError, match="outside"):
        capi.Solver.ams(b2p_ctx, Gs, nd_box["X"][:10])
    with pytest.raises(capi.B2PError):
        capi.Solver.amg(b2p_ctx, cycle_it=0)
    with pytest.raises(capi.B2PError):
        capi.Solver.jacobi(b2p_ctx).levels(0)


# ---------------------------------------------------------------------------------------------------- 9. CUDA graph
@pytest.mark.skipif(EMU, reason="stream capture needs the real device")
def test_ams_mult_replays_from_a_cuda_graph(b2p_ctx, nd_box):
    from palace_b200 import capi

    dev, _ = _ams(b2p_ctx, nd_box, cycle_it=2)
    n = nd_box["Ah"].shape[0]
    b = _dev(np.random.default_rng(11).standard_normal(n))
    y_eager = torch.zeros(n, dtype=torch.float64, device="cuda")
    capi.set_stream(b2p_ctx)
    dev.mult(b, y_eager)
    torch.cuda.synchronize()
    y = torch.zeros(n, dtype=torch.float64, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    try:
        with torch.cuda.graph(g, stream=s):
            capi.set_stream(b2p_ctx, s.cuda_stream)
            dev.mult(b, y)
    finally:
        capi.set_stream(b2p_ctx)
    y.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, y_eager)

"""The assembled coarse solver of complex systems (b2p_csolver_assembled, MfemWrapperSolver<ComplexOperator>): CSR assembly of the
non-symmetric hex block operators (Floquet mixed curl terms and their sums), the full assembly of both parts of a complex operator on
one pattern, the block-2 matrix [[Ar, Ai], [Ai, -Ar]] and Ar + Ai, the solver's two forms and the complex p-multigrid with it as
the coarse solver -- against the oracle's matrices and SciPy."""

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import pyoracle as O
from oracle import solvers as S
from palace_b200.host import assemble as asm
from palace_b200.host import coeff as cf
from palace_b200.host import hexmesh as hm
from palace_b200.host import hexspace as hs
from tests import common
from tests.test_cylinder_floquet_golden import cross_matrix

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
RTOL = 1e-12


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _host(t):
    return t.cpu().numpy().copy()


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def _srel(A, B):
    return spla.norm(sp.csr_matrix(A - B)) / max(spla.norm(sp.csr_matrix(B)), 1e-300)


def _mixed_ctx(kind, n_attr, seed=5):
    am, mc = cf.test_suite_coefficient(n_attr, "matrix")
    mc = mc + 0.3 * (np.random.default_rng(seed).random(mc.shape) - 0.5)
    if kind == O.ND_WEAKCURL:
        return cf.coeff_ctx(am, mc, a=-1.0)
    return cf.coeff_ctx(am, mc, a=1.0, transpose=True)


def floquet_problem(p):
    """The z-periodic hex box with the five terms of a Floquet system: curl-curl, the k-mass, i (weak curl + mixed curl) and a
    mass shift (K + 1.5 M: Hermitian positive definite)."""
    mesh = hm.box_mesh((3, 3, 3), (1.0, 0.8, 0.9), warp_amp=0.04, scramble_seed=11, periodic_z=True)
    prob = common.problem_on_mesh(mesh, p=p)
    kx = cross_matrix((0.0, 0.0, 0.4))
    am = np.array([0])
    terms = [(O.CURLCURL, cf.coeff_ctx(a=1.0)), (O.ND_MASS, cf.coeff_ctx(am, (kx.T @ kx)[None])),
             (O.ND_WEAKCURL, cf.coeff_ctx(am, kx[None], a=-1.0)), (O.ND_MIXEDCURL, cf.coeff_ctx(am, kx[None], transpose=True)),
             (O.ND_MASS, cf.coeff_ctx(a=1.0))]
    return prob, terms, [1.0, 1.0, 1j, 1j, 1.5]


def lossy_problem(p, w2=-2.0, tand=0.1):
    """A lossy cavity K - w2 (1 - i tan d) M with material tensors (w2 < 0: positive definite real part, as Chebyshev smoothing
    without auxiliary-space relaxation needs)."""
    prob = common.make_problem(n=(3, 3, 2), p=p, n_attr=3)
    terms = [(O.CURLCURL, common.coefficient(O.CURLCURL, 3)), (O.ND_MASS, common.coefficient(O.ND_MASS, 3))]
    return prob, terms, [1.0, -w2 * (1.0 - 1j * tand)]


def _parts_ref(prob, terms, coefs, space=None):
    """Ar, Ai of sum_t c_t M_t after elimination: DIAG_ONE for the real part, DIAG_ZERO for the imaginary part."""
    sp_ = prob.nd if space is None else space
    Z = sum(c * common.oracle_matrix(prob, k, b, space=sp_, eliminate=False) for c, (k, b) in zip(coefs, terms)).tocsr()
    return S.eliminate(Z.real, sp_.ess_dofs), S.eliminate(Z.imag, sp_.ess_dofs, diag_one=False)


def _complex_op(ctx, prob, terms, coefs, space=None, fine_ops=None):
    from palace_b200 import capi

    sp_ = prob.nd if space is None else space
    if fine_ops is None:
        geom = common.gpu_geom(ctx, prob)
        ops = [common.gpu_op(ctx, geom, prob, k, b, space=sp_) for k, b in terms]
    else:
        t = hs.tables_1d(sp_.p, prob.q1d)
        idx, ori = sp_.native_restriction()
        ops = [o.coarsen(sp_.p, sp_.ndofs, idx, ori, sp_.dof_map, t.Bo, t.Bc, t.Gc) for o in fine_ops]
    A = capi.ComplexOperator.par(ctx, sp_.ndofs, sp_.ndofs, ops, coefs, sp_.ess_dofs, diag_policy=1)
    A.local_ops = ops
    return A


def _assembled(ctx, complex_matrix, rel_tol=1e-12, max_it=1000, jacobi=True):
    """b2p_csolver_assembled over GMRES (+ Jacobi)."""
    from palace_b200 import capi

    inner = capi.Solver.krylov(ctx, capi.GMRES, rel_tol=rel_tol, max_it=max_it, max_dim=max_it)
    pc = capi.Solver.jacobi(ctx) if jacobi else None
    return capi.ComplexSolver.assembled(ctx, inner, pc, complex_matrix=complex_matrix)


def _matrix(solver, rows):
    rp, cl, vl = (_host(t) for t in solver.assembled_device_arrays())
    assert rp.size == rows + 1 and rp[-1] == cl.size == vl.size == solver.assembled_nnz()
    assert all(np.all(np.diff(cl[rp[i]:rp[i + 1]]) > 0) for i in range(rows))  # sorted, unique columns
    return sp.csr_matrix((vl, cl, rp), shape=(rows, rows))


def _split(B, n):
    """Ar, Ai from the block matrix [[Ar, Ai], [Ai, -Ar]], checking its other two blocks."""
    B = B.tocsr()
    Ar, Ai = B[:n, :n], B[:n, n:]
    assert (B[n:, :n] != Ai).nnz == 0 and (B[n:, n:] != -Ar).nnz == 0
    return Ar, Ai


# ---------------------------------------------------------------------------------------------------- 1. block operators in the CSR
@pytest.mark.parametrize("p", [1, 2, 3])
@pytest.mark.parametrize("which", ["weakcurl", "mixedcurl", "sum"])
def test_block_operator_csr_matches_oracle(b2p_ctx, p, which):
    """p = 1 runs the cross-check kernel, p = 2 and 3 nd_hex_apply6_kernel; 18 scrambled, warped elements (ragged batches)."""
    from palace_b200 import capi

    prob = common.make_problem(n=(3, 3, 2), p=p, n_attr=3)
    geom = common.gpu_geom(b2p_ctx, prob)
    if which == "sum":
        terms = [(O.CURLCURL, common.coefficient(O.CURLCURL, 3)), (O.ND_MASS, common.coefficient(O.ND_MASS, 3)),
                 (O.ND_WEAKCURL, _mixed_ctx(O.ND_WEAKCURL, 3)), (O.ND_MIXEDCURL, _mixed_ctx(O.ND_MIXEDCURL, 3, seed=8))]
        c = [1.0, -2.5, 0.7, 0.4]
        op = capi.Op.create_sum(b2p_ctx, [common.gpu_op(b2p_ctx, geom, prob, k, b) for k, b in terms], c)
    else:
        kind = O.ND_WEAKCURL if which == "weakcurl" else O.ND_MIXEDCURL
        terms, c = [(kind, _mixed_ctx(kind, 3))], [1.0]
        op = common.gpu_op(b2p_ctx, geom, prob, kind, terms[0][1])
    A_ref = sum(ci * common.oracle_matrix(prob, k, b, eliminate=False) for ci, (k, b) in zip(c, terms)).tocsr()
    assert _srel(A_ref, A_ref.T) > 1e-3  # not symmetric
    csr = capi.Csr(b2p_ctx, op)
    csr.assemble([op])
    A = csr.to_scipy()
    assert _srel(A, A_ref) < RTOL
    # A^T x from the CSR equals the transposed apply
    x = np.random.default_rng(p).standard_normal(prob.nd.ndofs)
    yt = torch.zeros(prob.nd.ndofs, dtype=torch.float64, device="cuda")
    op.apply_add_ex(1.0, _dev(x), yt, transpose=True)
    assert _rel(_host(yt), A.T @ x) < RTOL
    csr.close()


# ---------------------------------------------------------------------------------------------------- 2. complex full assembly
@pytest.mark.parametrize("problem,p", [("floquet", 1), ("floquet", 2), ("lossy", 1), ("lossy", 2)])
def test_complex_operator_parts_fused_and_term_by_term(b2p_ctx, problem, p, monkeypatch):
    prob, terms, coefs = (floquet_problem if problem == "floquet" else lossy_problem)(p)
    n = prob.nd.ndofs
    Ar_ref, Ai_ref = _parts_ref(prob, terms, coefs)
    got = {}
    for fused in ("1", "0"):
        monkeypatch.setenv("B2P_COMPLEX_FUSED", fused)
        A = _complex_op(b2p_ctx, prob, terms, coefs)
        s = _assembled(b2p_ctx, True)
        s.set_operator(A)
        Ar, Ai = _split(_matrix(s, 2 * n), n)
        assert _srel(Ar, Ar_ref) < RTOL and _srel(Ai, Ai_ref) < RTOL
        got[fused] = (Ar, Ai)
        # Ar + Ai on the same pattern
        s2 = _assembled(b2p_ctx, False)
        s2.set_operator(A)
        assert _srel(_matrix(s2, n), Ar_ref + Ai_ref) < RTOL
    for a, b in zip(got["1"], got["0"]):
        assert _srel(a, b) < 1e-14


def test_wrap_of_two_par_operators_assembles_the_same_parts(b2p_ctx):
    from palace_b200 import capi

    prob, terms, coefs = floquet_problem(1)
    nd = prob.nd
    n = nd.ndofs
    geom = common.gpu_geom(b2p_ctx, prob)
    ops = [common.gpu_op(b2p_ctx, geom, prob, k, b) for k, b in terms]
    Ar = capi.Operator.par(b2p_ctx, n, n, ops, [complex(c).real for c in coefs], nd.ess_dofs, diag_policy=1)
    Ai = capi.Operator.par(b2p_ctx, n, n, ops, [complex(c).imag for c in coefs], nd.ess_dofs, diag_policy=0)
    W = capi.ComplexOperator.wrap(b2p_ctx, Ar, Ai)
    s = _assembled(b2p_ctx, True)
    s.set_operator(W)
    Ar_ref, Ai_ref = _parts_ref(prob, terms, coefs)
    Br, Bi = _split(_matrix(s, 2 * n), n)
    assert _srel(Br, Ar_ref) < RTOL and _srel(Bi, Ai_ref) < RTOL
    # the real part alone: its matrix, not the block form
    s1 = _assembled(b2p_ctx, True)
    s1.set_operator(capi.ComplexOperator.wrap(b2p_ctx, Ar, None))
    assert _srel(_matrix(s1, n), Ar_ref) < RTOL


# ---------------------------------------------------------------------------------------------------- 3. kernels
@pytest.mark.parametrize("complex_matrix", [True, False])
def test_block2_spmv_and_diagonal_match_scipy(b2p_ctx, complex_matrix):
    """Jacobi as the inner solver applies the inverse diagonal; two GMRES steps without preconditioner give the minimiser of
    ||b - B x|| over span{b, B b}: both against SciPy on the explicit real matrix."""
    from palace_b200 import capi

    prob, terms, coefs = floquet_problem(1)
    n = prob.nd.ndofs
    Ar, Ai = _parts_ref(prob, terms, coefs)
    B = sp.bmat([[Ar, Ai], [Ai, -Ar]]).tocsr() if complex_matrix else (Ar + Ai).tocsr()
    A = _complex_op(b2p_ctx, prob, terms, coefs)
    rng = np.random.default_rng(3)
    br, bi = rng.standard_normal(n), rng.standard_normal(n)
    rhs = [np.concatenate([br, bi])] if complex_matrix else [br, bi]
    xr, xi = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda")

    def run(solver):
        solver.set_operator(A)
        solver.mult(_dev(br), _dev(bi), xr, xi)
        got = [np.concatenate([_host(xr), -_host(xi)])] if complex_matrix else [_host(xr), _host(xi)]
        return got

    d = B.diagonal()
    if complex_matrix:
        assert np.array_equal(d[n:], -d[:n])
    for g, b in zip(run(capi.ComplexSolver.assembled(b2p_ctx, capi.Solver.jacobi(b2p_ctx), None, complex_matrix=complex_matrix)), rhs):
        assert _rel(g, b / d) < RTOL
    for g, b in zip(run(_assembled(b2p_ctx, complex_matrix, rel_tol=0.0, max_it=2, jacobi=False)), rhs):
        V = np.stack([b, B @ b], axis=1)
        c = np.linalg.lstsq(B @ V, b, rcond=None)[0]
        assert _rel(g, V @ c) < 1e-10
    # the device arrays: the explicit matrix entry for entry
    s = _assembled(b2p_ctx, complex_matrix)
    s.set_operator(A)
    assert _srel(_matrix(s, B.shape[0]), B) < RTOL


# ---------------------------------------------------------------------------------------------------- 4. solver
@pytest.fixture(scope="module")
def box1(b2p_ctx):
    prob, terms, coefs = floquet_problem(1)
    Ar, Ai = _parts_ref(prob, terms, coefs)
    return dict(prob=prob, terms=terms, coefs=coefs, Ar=Ar, Ai=Ai, Z=(Ar + 1j * Ai).tocsc())


def test_block_mode_solves_the_complex_system(b2p_ctx, box1):
    prob, n = box1["prob"], box1["prob"].nd.ndofs
    A = _complex_op(b2p_ctx, prob, box1["terms"], box1["coefs"])
    s = _assembled(b2p_ctx, True)
    s.set_operator(A)
    rng = np.random.default_rng(5)
    b = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    xr, xi = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda")
    s.mult(_dev(b.real), _dev(b.imag), xr, xi)
    assert _rel(_host(xr) + 1j * _host(xi), spla.spsolve(box1["Z"], b)) < 1e-9


def test_sum_mode_applies_the_real_inverse_to_each_part(b2p_ctx, box1):
    prob, n = box1["prob"], box1["prob"].nd.ndofs
    A = _complex_op(b2p_ctx, prob, box1["terms"], box1["coefs"])
    s = _assembled(b2p_ctx, False)
    s.set_operator(A)
    Sm = (box1["Ar"] + box1["Ai"]).tocsc()
    rng = np.random.default_rng(6)
    br, bi = rng.standard_normal(n), rng.standard_normal(n)
    xr, xi = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda")
    s.mult(_dev(br), _dev(bi), xr, xi)
    assert _rel(_host(xr), spla.spsolve(Sm, br)) < 1e-9
    assert _rel(_host(xi), spla.spsolve(Sm, bi)) < 1e-9


@pytest.mark.parametrize("complex_matrix", [True, False])
def test_initial_guess_is_honoured(b2p_ctx, box1, complex_matrix):
    """Three inner GMRES steps do not solve the system from zero; from the solution as the initial guess they keep it."""
    prob, n = box1["prob"], box1["prob"].nd.ndofs
    A = _complex_op(b2p_ctx, prob, box1["terms"], box1["coefs"])
    s = _assembled(b2p_ctx, complex_matrix, max_it=3)
    s.set_operator(A)
    rng = np.random.default_rng(8)
    b = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    if complex_matrix:
        x = spla.spsolve(box1["Z"], b)
    else:
        Sm = (box1["Ar"] + box1["Ai"]).tocsc()
        x = spla.spsolve(Sm, b.real) + 1j * spla.spsolve(Sm, b.imag)
    for guess in (False, True):
        s.set_initial_guess(guess)
        xr, xi = _dev(x.real), _dev(x.imag)
        s.mult(_dev(b.real), _dev(b.imag), xr, xi)
        err = _rel(_host(xr) + 1j * _host(xi), x)
        assert (err < 1e-9) if guess else (err > 1e-6), (guess, err)


def test_reassembly_after_new_coefficients_keeps_the_pattern(b2p_ctx, box1):
    prob, terms, n = box1["prob"], box1["terms"], box1["prob"].nd.ndofs
    A = _complex_op(b2p_ctx, prob, terms, box1["coefs"])
    for complex_matrix in (True, False):
        s = _assembled(b2p_ctx, complex_matrix)
        s.set_operator(A)
        rp0 = s.assembled_device_arrays()[0].data_ptr()
        coefs2 = [1.0, 1.0, 0.5j, 0.5j, 2.0 + 0.3j]
        A.set_coefficients(coefs2)
        s.set_operator(A)
        assert s.assembled_device_arrays()[0].data_ptr() == rp0  # no new symbolic phase
        Ar, Ai = _parts_ref(prob, terms, coefs2)
        if complex_matrix:
            Br, Bi = _split(_matrix(s, 2 * n), n)
            assert _srel(Br, Ar) < RTOL and _srel(Bi, Ai) < RTOL
        else:
            assert _srel(_matrix(s, n), Ar + Ai) < RTOL
        A.set_coefficients(box1["coefs"])


def test_nnz_through_the_multigrid_and_error_paths(b2p_ctx):
    from palace_b200 import capi

    prob, terms, coefs = floquet_problem(2)
    nd1 = hs.build_nd_space(prob.mesh, prob.topo, 1)
    A2 = _complex_op(b2p_ctx, prob, terms, coefs)
    A1 = _complex_op(b2p_ctx, prob, terms, coefs, space=nd1, fine_ops=A2.local_ops)
    P = [common.gpu_interp(b2p_ctx, nd1, prob.nd, asm.nd_prolongation_comps(1, 2))]
    nnz = {}
    for complex_matrix in (True, False):
        coarse = _assembled(b2p_ctx, complex_matrix)
        assert coarse.assembled_nnz() == -1
        mg = capi.ComplexSolver.gmg(b2p_ctx, coarse, P, None, cycle_it=1, smooth_it=1, cheby_order=4)
        assert mg.assembled_nnz() == -1
        mg.gmg_set_operators([A1, A2])
        nnz[complex_matrix] = mg.assembled_nnz()
        assert nnz[complex_matrix] == _host(mg.assembled_device_arrays()[0])[-1] > 0
    assert nnz[True] == 4 * nnz[False]
    # parts that cannot be assembled: the assembled matrices behind the operator interface
    geom = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, geom, prob, O.ND_MASS, cf.coeff_ctx(a=1.0))
    csr = capi.Csr(b2p_ctx, op)
    csr.assemble([op])
    W = capi.ComplexOperator.wrap(b2p_ctx, capi.Operator.from_csr(b2p_ctx, csr), capi.Operator.from_csr(b2p_ctx, csr))
    s = _assembled(b2p_ctx, True)
    with pytest.raises(capi.B2PError, match="must be ParOperators"):
        s.set_operator(W)
    assert s.assembled_nnz() == -1
    with pytest.raises(capi.B2PError, match="before set_operator"):
        s.assembled_device_arrays()
    csr.close()


# ---------------------------------------------------------------------------------------------------- 5. end to end
def _fgmres_mg(ctx, prob, terms, coefs, orders, complex_matrix):
    from palace_b200 import capi

    nd = {p: hs.build_nd_space(prob.mesh, prob.topo, p) for p in orders}
    top = orders[-1]
    A = {top: _complex_op(ctx, prob, terms, coefs)}
    for p in reversed(orders[:-1]):
        A[p] = _complex_op(ctx, prob, terms, coefs, space=nd[p], fine_ops=A[top].local_ops)
    P = [common.gpu_interp(ctx, nd[a], nd[b], asm.nd_prolongation_comps(a, b)) for a, b in zip(orders[:-1], orders[1:])]
    coarse = _assembled(ctx, complex_matrix, rel_tol=1e-12)
    mg = capi.ComplexSolver.gmg(ctx, coarse, P, None, cycle_it=1, smooth_it=1, cheby_order=4)
    mg.gmg_set_operators([A[p] for p in orders])
    Ks = capi.ComplexSolver.krylov(ctx, capi.FGMRES, rel_tol=1e-10, max_it=200, max_dim=200)
    Ks.set_operator(A[top])
    Ks.set_preconditioner(mg)
    n = nd[top].ndofs
    rng = np.random.default_rng(31)
    b = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    b[nd[top].ess_dofs] = 0.0
    zr, zi = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda")
    Ks.mult(_dev(b.real), _dev(b.imag), zr, zi)
    Ar, Ai = _parts_ref(prob, terms, coefs)
    x = spla.spsolve((Ar + 1j * Ai).tocsc(), b)
    return Ks.stats(), _rel(_host(zr) + 1j * _host(zi), x)


def test_fgmres_with_assembled_block_coarse_solver_on_the_periodic_box(b2p_ctx):
    from palace_b200 import capi

    capi.set_stream(b2p_ctx)
    prob, terms, coefs = floquet_problem(3)
    st, err = _fgmres_mg(b2p_ctx, prob, terms, coefs, [1, 2, 3], True)
    print("periodic box, FGMRES + complex p-multigrid {1, 2, 3}, assembled block coarse solver:", st, "error", err)
    assert st["converged"] and err < 1e-8, (st, err)


def test_fgmres_with_assembled_sum_coarse_solver_on_a_lossy_cavity(b2p_ctx):
    from palace_b200 import capi

    capi.set_stream(b2p_ctx)
    prob, terms, coefs = lossy_problem(2)
    st, err = _fgmres_mg(b2p_ctx, prob, terms, coefs, [1, 2], False)
    print("lossy cavity p = 2, FGMRES + complex p-multigrid {1, 2}, assembled Ar + Ai coarse solver:", st, "error", err)
    assert st["converged"] and err < 1e-8, (st, err)

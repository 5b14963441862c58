"""GPU parity of the complex apply on the CTA-per-batch kernel (nd_hex_apply7_kernel<..., CPLX>): one pass over the geometry for
every term and both parts of a split complex vector.

- Symmetric kinds (curl-curl, mass, curl-curl + mass) at p = 4, 5, 6: sums of two or more terms.
- Floquet block sums (the mixed curl kinds fused with curl-curl and mass) at p = 2 ... 6, on the z-periodic box.

Each is checked against the term-by-term path (B2P_COMPLEX_FUSED=0, four real applies per term) and against complex arithmetic on
the oracle's assembled matrices, at 1e-12 relative (FP64, different summation order)."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

from oracle import pyoracle as O
from palace_b200.host import assemble as asm
from palace_b200.host import hexspace as hs
from tests import common
from oracle import solvers as S
from palace_b200.host import hexmesh as hm
from tests.test_zzcomplex_assembled_gpu import _assembled, _matrix, _split, _srel, floquet_problem

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
RTOL = 1e-12


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _host(yr, yi):
    return yr.cpu().numpy() + 1j * yi.cpu().numpy()


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def _elim(Z, ess, diag_policy):
    Z = Z.tolil()
    Z[ess, :] = 0
    Z[:, ess] = 0
    Z[ess, ess] = 1.0 if diag_policy == 1 else 0.0
    return Z.tocsr()


def _terms(which, n_attr):
    mk = lambda kind, **kw: (kind, common.coefficient(kind, n_attr, **kw))
    return {
        "K+M lossy": [(mk(O.CURLCURL, coeff_type="const"), 1.0 + 0.0j), (mk(O.ND_MASS, coeff_type="matrix"), -9.0 * (1 - 0.05j))],
        "four terms": [(mk(O.CURLCURL, coeff_type="matrix"), 1.0 + 0.0j), (mk(O.ND_MASS, coeff_type="matrix", a_mass=1.7), -2.5 + 0.4j),
                       (mk(O.ND_MASS, coeff_type="scalar", a_mass=0.3), 1.3j), (mk(O.CURLCURL_MASS, coeff_type="matrix"), 0.2 - 0.1j)],
        "real coefficients": [(mk(O.CURLCURL_MASS, coeff_type="matrix"), 0.7 + 0.0j), (mk(O.ND_MASS, coeff_type="const"), 2.0 + 0.0j)],
        # K - w^2 (1 - i tan d) M + i w C, C a second (boundary-like) mass term
        "K+M+C": [(mk(O.CURLCURL, coeff_type="matrix"), 1.0 + 0.0j), (mk(O.ND_MASS, coeff_type="matrix"), -4.0 * (1 - 0.02j)),
                  (mk(O.ND_MASS, coeff_type="scalar", a_mass=0.3), 2.0j)],
    }[which]


def _build(ctx, prob, spec):
    geom = common.gpu_geom(ctx, prob)
    ops = [common.gpu_op(ctx, geom, prob, kind, blob) for (kind, blob), _ in spec]
    mats = [common.oracle_matrix(prob, kind, blob, eliminate=False) for (kind, blob), _ in spec]
    return ops, [c for _, c in spec], mats


def _pair(ctx, monkeypatch, nd, ops, coefs, diag_policy=1):
    """The same complex sum term by term and on the default route."""
    from palace_b200 import capi

    monkeypatch.setenv("B2P_COMPLEX_FUSED", "0")
    A_terms = capi.ComplexOperator.par(ctx, nd.ndofs, nd.ndofs, ops, coefs, nd.ess_dofs, diag_policy)
    monkeypatch.setenv("B2P_COMPLEX_FUSED", "1")
    A = capi.ComplexOperator.par(ctx, nd.ndofs, nd.ndofs, ops, coefs, nd.ess_dofs, diag_policy)
    return A_terms, A


def _mult_both(A, x):
    xr, xi = _dev(x.real), _dev(x.imag)
    yr, yi = torch.full_like(xr, 3.0), torch.full_like(xr, -2.0)
    A.mult(xr, xi, yr, yi)
    hr, hi = torch.full_like(xr, 1.0), torch.empty_like(xr)
    A.mult_hermitian_transpose(xr, xi, hr, hi)
    return _host(yr, yi), _host(hr, hi)


# odd element counts: a ragged last batch at p = 5 (two elements per batch); few elements at p = 5, 6, where the oracle's
# element matrices are expensive
MESH = {4: (3, 1, 3), 5: (3, 1, 1), 6: (3, 1, 1)}


def _floquet(p, q1d=None):
    """The Floquet system of floquet_problem on a smaller z-periodic box (three layers, the fewest the identification allows)."""
    _, terms, coefs = floquet_problem(1)
    n = (2, 1, 3) if p <= 4 else (1, 1, 3)
    mesh = hm.box_mesh(n, (1.0, 0.8, 0.9), warp_amp=0.04, scramble_seed=11, periodic_z=True)
    return common.problem_on_mesh(mesh, p=p, q1d=q1d), terms, coefs


# ---------------------------------------------------------------------------------------------------- 1. symmetric sums, p = 4 ... 6
@pytest.mark.parametrize("which", ["K+M lossy", "four terms", "real coefficients", "K+M+C"])
@pytest.mark.parametrize("p", [4, 5, 6])
def test_symmetric_sum_one_pass(b2p_ctx, monkeypatch, p, which):
    n_attr = 3
    prob = common.make_problem(n=MESH[p], p=p, n_attr=n_attr)
    nd = prob.nd
    ops, coefs, mats = _build(b2p_ctx, prob, _terms(which, n_attr))
    Z = sum(c * M for c, M in zip(coefs, mats))
    x = np.random.default_rng(p).random(nd.ndofs) + 1j * np.random.default_rng(p + 10).random(nd.ndofs)
    for diag_policy in (1, 0):
        A_terms, A = _pair(b2p_ctx, monkeypatch, nd, ops, coefs, diag_policy)
        assert A_terms.fused_path() == 0 and A.fused_path() == 3
        got, ref = _mult_both(A, x), _mult_both(A_terms, x)
        assert A.fused_applies() == 2 and A_terms.fused_applies() == 0
        Ze = _elim(Z, nd.ess_dofs, diag_policy)
        for g, r, o in zip(got, ref, (Ze @ x, Ze.conj().T @ x)):
            assert _rel(g, r) < RTOL
            assert _rel(g, o) < RTOL


# ---------------------------------------------------------------------------------------------------- 2. accumulating applies
@pytest.mark.parametrize("p", [4, 6])
def test_add_mult_real_and_complex_scalar(b2p_ctx, monkeypatch, p):
    prob = common.make_problem(n=MESH[p], p=p, n_attr=3)
    nd = prob.nd
    ops, coefs, mats = _build(b2p_ctx, prob, _terms("K+M+C", 3))
    _, A = _pair(b2p_ctx, monkeypatch, nd, ops, coefs)
    assert A.fused_path() == 3
    Ze = _elim(sum(c * M for c, M in zip(coefs, mats)), nd.ess_dofs, 1)
    rng = np.random.default_rng(4)
    x = rng.random(nd.ndofs) + 1j * rng.random(nd.ndofs)
    y0 = rng.random(nd.ndofs) + 1j * rng.random(nd.ndofs)
    for a in (-1.0, 0.5 - 0.75j):
        yr, yi = _dev(y0.real), _dev(y0.imag)
        A.add_mult(_dev(x.real), _dev(x.imag), yr, yi, a)
        assert _rel(_host(yr, yi), y0 + a * (Ze @ x)) < RTOL


# ---------------------------------------------------------------------------------------------------- 3. frequency sweep
def test_frequency_sweep_with_a_real_point(b2p_ctx, monkeypatch):
    """New coefficients in place; the last set has every c_t^i = 0 (the parts are not coupled)."""
    prob = common.make_problem(n=MESH[4], p=4, n_attr=3)
    nd = prob.nd
    ops, _, mats = _build(b2p_ctx, prob, _terms("K+M+C", 3))
    sweep = [[1.0, -1.0 * (1 - 0.02j), 1.0j], [1.0, -6.25 * (1 - 0.02j), 2.5j], [1.0, -0.16, 0.0]]
    A_terms, A = _pair(b2p_ctx, monkeypatch, nd, ops, sweep[0])
    x = np.random.default_rng(3).random(nd.ndofs) + 1j * np.random.default_rng(5).random(nd.ndofs)
    for coefs in sweep:
        A.set_coefficients(coefs)
        A_terms.set_coefficients(coefs)
        Ze = _elim(sum(c * M for c, M in zip(coefs, mats)), nd.ess_dofs, 1)
        got, ref = _mult_both(A, x), _mult_both(A_terms, x)
        for g, r, o in zip(got, ref, (Ze @ x, Ze.conj().T @ x)):
            assert _rel(g, r) < RTOL and _rel(g, o) < RTOL
    assert A.fused_path() == 3 and A.fused_applies() == 6


# ---------------------------------------------------------------------------------------------------- 4. Floquet block sums
@pytest.mark.parametrize("p", [2, 3, 4, 5, 6])
def test_floquet_block_sum_one_pass(b2p_ctx, monkeypatch, p):
    prob, terms, coefs = _floquet(p)
    nd = prob.nd
    ops, coefs, mats = _build(b2p_ctx, prob, list(zip(terms, coefs)))
    A_terms, A = _pair(b2p_ctx, monkeypatch, nd, ops, coefs)
    assert A_terms.fused_path() == 0 and A.fused_path() == 3
    Z = sum(c * M for c, M in zip(coefs, mats)).tocsr()
    Ze = _elim(Z, nd.ess_dofs, 1)
    x = np.random.default_rng(p).standard_normal(nd.ndofs) + 1j * np.random.default_rng(p + 1).standard_normal(nd.ndofs)
    got, ref = _mult_both(A, x), _mult_both(A_terms, x)
    for g, r, o in zip(got, ref, (Ze @ x, Ze.conj().T @ x)):
        assert _rel(g, r) < RTOL and _rel(g, o) < RTOL
    assert A.fused_applies() == 2
    # the assembled coarse solver still assembles from S_re / S_im: DIAG_ONE rows in the real part, DIAG_ZERO in the imaginary part
    Ar_ref, Ai_ref = S.eliminate(Z.real, nd.ess_dofs), S.eliminate(Z.imag, nd.ess_dofs, diag_one=False)
    s = _assembled(b2p_ctx, True)
    s.set_operator(A)
    Ar, Ai = _split(_matrix(s, 2 * nd.ndofs), nd.ndofs)
    assert _srel(Ar, Ar_ref) < RTOL and _srel(Ai, Ai_ref) < RTOL


# ---------------------------------------------------------------------------------------------------- 5. fallbacks
@pytest.mark.parametrize("case", ["symmetric q1d = p + 2", "block q1d = p + 2", "block p = 1"])
def test_fallback_routes(b2p_ctx, monkeypatch, case):
    if case.startswith("symmetric"):
        prob = common.make_problem(n=(2, 1, 2), p=4, q1d=6, n_attr=3)
        spec, route = _terms("K+M lossy", 3), 0
    else:
        prob, terms, coefs = _floquet(4, q1d=6) if "q1d" in case else _floquet(1)
        spec, route = list(zip(terms, coefs)), 1
    nd = prob.nd
    ops, coefs, mats = _build(b2p_ctx, prob, spec)
    _, A = _pair(b2p_ctx, monkeypatch, nd, ops, coefs)
    assert A.fused_path() == route
    Ze = _elim(sum(c * M for c, M in zip(coefs, mats)), nd.ess_dofs, 1)
    x = np.random.default_rng(9).standard_normal(nd.ndofs) + 1j * np.random.default_rng(8).standard_normal(nd.ndofs)
    got = _mult_both(A, x)
    assert _rel(got[0], Ze @ x) < RTOL and _rel(got[1], Ze.conj().T @ x) < RTOL


# ---------------------------------------------------------------------------------------------------- 6. end to end
def _fgmres_pmg(ctx, prob, spec, orders):
    """FGMRES preconditioned with a complex p-multigrid (Chebyshev smoothing, coarse levels p-coarsened from the fine operators)."""
    from palace_b200 import capi

    capi.set_stream(ctx)
    p = orders[-1]
    nd = {q: hs.build_nd_space(prob.mesh, prob.topo, q) for q in orders}
    geom = common.gpu_geom(ctx, prob)
    fine = [common.gpu_op(ctx, geom, prob, k, b) for (k, b), _ in spec]
    coefs = [c for _, c in spec]
    A = {p: capi.ComplexOperator.par(ctx, nd[p].ndofs, nd[p].ndofs, fine, coefs, nd[p].ess_dofs, 1)}
    keep = [fine]
    for q in orders[:-1]:
        t = hs.tables_1d(q, prob.q1d)
        idx, ori = nd[q].native_restriction()
        ops = [o.coarsen(q, nd[q].ndofs, idx, ori, nd[q].dof_map, t.Bo, t.Bc, t.Gc) for o in fine]
        keep.append(ops)
        A[q] = capi.ComplexOperator.par(ctx, nd[q].ndofs, nd[q].ndofs, ops, coefs, nd[q].ess_dofs, 1)
    P = [common.gpu_interp(ctx, nd[a], nd[b], asm.nd_prolongation_comps(a, b)) for a, b in zip(orders[:-1], orders[1:])]
    coarse = capi.ComplexSolver.krylov(ctx, 1, rel_tol=1e-13, max_it=1000, max_dim=1000)
    mg = capi.ComplexSolver.gmg(ctx, coarse, P, None, cycle_it=1, smooth_it=1, cheby_order=4)
    mg.gmg_set_operators([A[q] for q in orders])
    Ks = capi.ComplexSolver.krylov(ctx, capi.FGMRES, rel_tol=1e-10, max_it=400, max_dim=400)
    Ks.set_operator(A[p])
    Ks.set_preconditioner(mg)
    n = nd[p].ndofs
    rng = np.random.default_rng(31)
    b = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    b[nd[p].ess_dofs] = 0.0
    zr, zi = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda")
    Ks.mult(_dev(b.real), _dev(b.imag), zr, zi)
    return Ks.stats(), _host(zr, zi), b, A[p].fused_path(), nd[p]


def test_fgmres_with_complex_p_multigrid_on_a_lossy_p4_box(b2p_ctx, monkeypatch):
    prob = common.make_problem(n=(3, 2, 2), p=4, n_attr=3)
    spec = [((O.CURLCURL, common.coefficient(O.CURLCURL, 3)), 1.0 + 0.0j),
            ((O.ND_MASS, common.coefficient(O.ND_MASS, 3)), 10.0 * (1.0 - 0.1j))]
    out = {}
    for fused in ("0", "1"):
        monkeypatch.setenv("B2P_COMPLEX_FUSED", fused)
        out[fused] = _fgmres_pmg(b2p_ctx, prob, spec, [1, 2, 4])
    (st0, z0, b, path0, nd), (st1, z1, _, path1, _) = out["0"], out["1"]
    print("FGMRES + complex p-multigrid:", st0, st1)
    assert path0 == 0 and path1 == 3
    assert st1["converged"] and st1["its"] == st0["its"], (st0, st1)
    Z = _elim(sum(c * common.oracle_matrix(prob, k, blob, eliminate=False) for (k, blob), c in spec), nd.ess_dofs, 1)
    assert _rel(z1, spla.spsolve(Z.tocsc(), b)) < 1e-8

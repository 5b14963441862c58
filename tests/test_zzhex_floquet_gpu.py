"""The Floquet-periodic mixed curl terms on hexahedra through the sum-factorised path: b2p_op_create with B2P_ND_WEAKCURL /
B2P_ND_MIXEDCURL (block operators: the per-element tensors {Cm, Ck, Cw, Cx} and their transposed block), their sums with
curl-curl and mass terms (one block operator), the fused ParOperator and ComplexParOperator over them, and a complex
p-multigrid on the periodic hex box -- against the oracle, the dense-table operators of the same kinds and SciPy."""

import numpy as np
import pytest
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
MIXED = [O.ND_WEAKCURL, O.ND_MIXEDCURL]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def mixed_ctx(kind, n_attr, coeff_type="matrix", seed=5):
    """Context of a mixed curl integrator as Palace builds it: a = -1 for the weak curl, transposed matrices for the curl
    (non-symmetric per-material matrices, or scalars)."""
    am, mc = cf.test_suite_coefficient(n_attr, coeff_type)
    if coeff_type == "matrix":
        mc = mc + 0.3 * (np.random.default_rng(seed).random(mc.shape) - 0.5)
    if kind == O.ND_WEAKCURL:
        return cf.coeff_ctx(am, mc, a=-1.0)
    return cf.coeff_ctx(am, mc, a=1.0, transpose=True)


def dense_op(ctx, prob, kind, blob):
    from palace_b200 import capi

    geom = capi.Geom.general(ctx, prob.qdata_ref)
    interp, curl, _ = O.nd_hex_tables(prob.nd.p, prob.q1d)
    idx, ori = prob.nd.native_restriction()
    return capi.Op.create_dense(ctx, geom, kind, prob.nd.ndofs, idx, ori, interp, curl, blob)


CASES = [(p, p + 1) for p in range(1, 7)] + [(2, 4)]


@pytest.mark.parametrize("coeff_type", ["matrix", "scalar"])
@pytest.mark.parametrize("p,q1d", CASES)
@pytest.mark.parametrize("kind", MIXED)
def test_mixed_kind_on_hexes_matches_oracle_and_dense_operator(b2p_ctx, kind, p, q1d, coeff_type):
    n = (3, 3, 2) if p <= 3 else (3, 2, 2)  # 18 / 12 warped, scrambled elements: ragged element batches
    prob = common.make_problem(n=n, p=p, q1d=q1d, n_attr=3)
    blob = mixed_ctx(kind, 3, coeff_type)
    geom = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, geom, prob, kind, blob)
    nd = prob.nd
    ndofs = nd.ndofs
    rng = np.random.default_rng(10 * p + q1d)
    x, y0 = rng.standard_normal(ndofs), rng.standard_normal(ndofs)
    A = common.oracle_matrix(prob, kind, blob, eliminate=False).tocsr()
    y_ref = common.oracle_apply(prob, kind, blob, x)
    assert _rel(A @ x, y_ref) < RTOL
    yd = torch.full((ndofs,), 3.0, dtype=torch.float64, device="cuda")
    op.apply(_dev(x), yd)
    y = yd.cpu().numpy()
    assert _rel(y, y_ref) < RTOL
    # the dense-table operator of the same kind
    yq = torch.zeros(ndofs, dtype=torch.float64, device="cuda")
    dense_op(b2p_ctx, prob, kind, blob).apply(_dev(x), yq)
    assert _rel(y, yq.cpu().numpy()) < RTOL
    # alpha; the default kernel (nd_hex_apply6_kernel at p = 2, 3, nd_hex_apply7_kernel at p = 4-6, both at q1d = p + 1) against
    # the cross-check kernel (B2P_APPLY_SIMPLE_KERNEL, which every other block operator runs on)
    for simple in (False, True):
        ya = _dev(y0)
        op.apply_add_ex(-0.75, _dev(x), ya, simple_kernel=simple)
        assert _rel(ya.cpu().numpy(), y0 - 0.75 * y_ref) < RTOL
        if simple:
            assert np.abs(ya.cpu().numpy() - y_prev).max() <= 1e-14 * np.abs(y_prev).max()
        y_prev = ya.cpu().numpy()
    # transpose: A^T of the oracle matrix
    yt = _dev(y0)
    op.apply_add_ex(1.0, _dev(x), yt, transpose=True)
    assert _rel(yt.cpu().numpy(), y0 + A.T @ x) < RTOL
    # masked: essential dofs eliminated on both sides (transposed too)
    ess = nd.ess_dofs
    op.set_essential(ess)
    xm = x.copy()
    xm[ess] = 0.0
    for tr in (False, True):
        ym = (A.T if tr else A) @ xm
        ym[ess] = 0.0
        yd = _dev(y0)
        op.apply_add_ex(0.5, _dev(x), yd, masked=True, transpose=tr)
        assert _rel(yd.cpu().numpy(), y0 + 0.5 * ym) < RTOL
    # owned | ghost split over two element ranges
    n_owned = ndofs // 2
    ne = prob.mesh.ne
    xd = _dev(x)
    yo = torch.zeros(n_owned, dtype=torch.float64, device="cuda")
    yg = torch.zeros(ndofs - n_owned, dtype=torch.float64, device="cuda")
    for e0, ec in ((0, ne // 3 + 1), (ne // 3 + 1, ne - ne // 3 - 1)):
        op.apply_add_split(1.0, xd[:n_owned].contiguous(), xd[n_owned:].contiguous(), yo, yg, n_owned, e0, ec)
    assert _rel(np.concatenate([yo.cpu().numpy(), yg.cpu().numpy()]), y_ref) < RTOL
    # the two-vector apply falls back to two applies
    y0d, y1d = torch.zeros(ndofs, dtype=torch.float64, device="cuda"), torch.zeros(ndofs, dtype=torch.float64, device="cuda")
    op.apply_add_pair(1.0, _dev(x), _dev(y0), y0d, y1d)
    assert _rel(y0d.cpu().numpy(), y_ref) < RTOL and _rel(y1d.cpu().numpy(), A @ y0) < RTOL
    # coefficient block of 4 tensors in the byte model
    assert op.algorithmic_bytes() == 16 * ndofs + ne * (4 * ((nd.P + 3) & ~3) + 80 * q1d ** 3 + 288)


@pytest.mark.parametrize("p", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", MIXED)
def test_mixed_kind_diagonal_and_new_coefficient(b2p_ctx, kind, p):
    prob = common.make_problem(n=(3, 2, 2), p=p, n_attr=3)
    geom = common.gpu_geom(b2p_ctx, prob)
    blob = mixed_ctx(kind, 3)
    op = common.gpu_op(b2p_ctx, geom, prob, kind, blob)
    n = prob.nd.ndofs
    dd = torch.zeros(n, dtype=torch.float64, device="cuda")
    op.diag_add(dd)
    d_ref = common.oracle_diag(prob, kind, blob)
    assert np.abs(dd.cpu().numpy() - d_ref).max() < RTOL * np.abs(d_ref).max()
    # b2p_op_set_coeff refills the block (and its transpose) in place
    blob2 = mixed_ctx(kind, 3, seed=9)
    op.set_coeff(blob2)
    x = np.random.default_rng(4).standard_normal(n)
    A2 = common.oracle_matrix(prob, kind, blob2, eliminate=False)
    for tr in (False, True):
        yd = torch.zeros(n, dtype=torch.float64, device="cuda")
        op.apply_add_ex(1.0, _dev(x), yd, transpose=tr)
        assert _rel(yd.cpu().numpy(), (A2.T if tr else A2) @ x) < RTOL


@pytest.mark.parametrize("kind", MIXED)
def test_coarsened_mixed_kind_matches_oracle_at_the_fine_quadrature(b2p_ctx, kind):
    prob = common.make_problem(n=(3, 2, 2), p=3, n_attr=3)
    geom = common.gpu_geom(b2p_ctx, prob)
    blob = mixed_ctx(kind, 3)
    fine = common.gpu_op(b2p_ctx, geom, prob, kind, blob)
    for pc in (1, 2):
        nd_c = hs.build_nd_space(prob.mesh, prob.topo, pc)
        t = hs.tables_1d(pc, prob.q1d)
        idx, ori = nd_c.native_restriction()
        coarse = fine.coarsen(pc, nd_c.ndofs, idx, ori, nd_c.dof_map, t.Bo, t.Bc, t.Gc)
        x = np.random.default_rng(pc).standard_normal(nd_c.ndofs)
        A = common.oracle_matrix(prob, kind, blob, space=nd_c, eliminate=False)
        for tr in (False, True):
            yd = torch.zeros(nd_c.ndofs, dtype=torch.float64, device="cuda")
            coarse.apply_add_ex(1.0, _dev(x), yd, transpose=tr)
            assert _rel(yd.cpu().numpy(), (A.T if tr else A) @ x) < RTOL


def floquet_terms(k):
    """The four Floquet terms of a unit-material periodic model (floquet_matrices of test_cylinder_floquet_golden.py):
    kinds and contexts of curl-curl, the k-mass, the weak curl and the mixed curl."""
    kx = cross_matrix(k)
    am = np.array([0])
    return [(O.CURLCURL, cf.coeff_ctx(a=1.0)), (O.ND_MASS, cf.coeff_ctx(am, (kx.T @ kx)[None])),
            (O.ND_WEAKCURL, cf.coeff_ctx(am, kx[None], a=-1.0)), (O.ND_MIXEDCURL, cf.coeff_ctx(am, kx[None], transpose=True))]


def test_sum_of_floquet_terms_is_one_block_operator(b2p_ctx):
    from palace_b200 import capi

    prob = common.make_problem(n=(3, 3, 2), p=3, n_attr=3)
    geom = common.gpu_geom(b2p_ctx, prob)
    nd = prob.nd
    n = nd.ndofs
    # material-dependent tensors in every term
    terms = [(O.CURLCURL, common.coefficient(O.CURLCURL, 3)), (O.ND_MASS, common.coefficient(O.ND_MASS, 3)),
             (O.ND_WEAKCURL, mixed_ctx(O.ND_WEAKCURL, 3)), (O.ND_MIXEDCURL, mixed_ctx(O.ND_MIXEDCURL, 3))]
    ops = [common.gpu_op(b2p_ctx, geom, prob, k, b) for k, b in terms]
    mats = [common.oracle_matrix(prob, k, b, eliminate=False) for k, b in terms]
    c = [1.0, -2.5, 0.7, 0.7]
    Asum = sum(ci * M for ci, M in zip(c, mats)).tocsr()
    S_op = capi.Op.create_sum(b2p_ctx, ops, c)
    rng = np.random.default_rng(12)
    x = rng.standard_normal(n)
    for tr in (False, True):
        y_terms = torch.zeros(n, dtype=torch.float64, device="cuda")
        for ci, o in zip(c, ops):
            o.apply_add_ex(ci, _dev(x), y_terms, transpose=tr)
        ys = torch.zeros(n, dtype=torch.float64, device="cuda")
        S_op.apply_add_ex(1.0, _dev(x), ys, transpose=tr)
        assert _rel(ys.cpu().numpy(), y_terms.cpu().numpy()) < RTOL
        assert _rel(ys.cpu().numpy(), (Asum.T if tr else Asum) @ x) < RTOL
    dd = torch.zeros(n, dtype=torch.float64, device="cuda")
    S_op.diag_add(dd)
    assert _rel(dd.cpu().numpy(), Asum.diagonal()) < RTOL
    # the ParOperator over the term list fuses by itself; Mult and MultTranspose against the eliminated oracle sum
    A = capi.Operator.par(b2p_ctx, n, n, ops, c, nd.ess_dofs, diag_policy=1)
    assert A.is_fused()
    Ael = S.eliminate(Asum, nd.ess_dofs)
    y = torch.empty(n, dtype=torch.float64, device="cuda")
    A.mult(_dev(x), y)
    assert _rel(y.cpu().numpy(), Ael @ x) < RTOL
    A.mult_transpose(_dev(x), y)
    assert _rel(y.cpu().numpy(), Ael.T @ x) < RTOL
    # new coefficients in place
    c2 = [0.5, 1.5, -0.2, 0.3]
    A.set_coefficients(c2)
    Ael2 = S.eliminate(sum(ci * M for ci, M in zip(c2, mats)).tocsr(), nd.ess_dofs)
    A.mult(_dev(x), y)
    assert _rel(y.cpu().numpy(), Ael2 @ x) < RTOL
    A.mult_transpose(_dev(x), y)
    assert _rel(y.cpu().numpy(), Ael2.T @ x) < RTOL


@pytest.fixture(scope="module")
def periodic(b2p_ctx):
    """Floquet system on the periodic hex box: terms, their oracle matrices and Z = K_r + i K_i - sigma M (PEC x / y walls)."""
    mesh = hm.box_mesh((3, 3, 3), (1.0, 0.8, 0.9), warp_amp=0.04, scramble_seed=11, periodic_z=True)
    prob = common.problem_on_mesh(mesh, p=3)
    terms = floquet_terms((0.0, 0.0, 0.4)) + [(O.ND_MASS, cf.coeff_ctx(a=1.0))]
    sigma = -1.5
    coefs = [1.0, 1.0, 1j, 1j, -sigma]
    return dict(prob=prob, terms=terms, coefs=coefs,
                mats=[common.oracle_matrix(prob, k, b, eliminate=False) for k, b in terms])


def _elim(Z, ess):
    Z = Z.tolil()
    Z[ess, :] = 0
    Z[:, ess] = 0
    Z[ess, ess] = 1.0
    return Z.tocsr()


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


@pytest.mark.parametrize("fused_env", ["1", "0"])
def test_complex_floquet_operator_on_the_periodic_box(b2p_ctx, periodic, fused_env, monkeypatch):
    prob, terms, coefs = periodic["prob"], periodic["terms"], periodic["coefs"]
    monkeypatch.setenv("B2P_COMPLEX_FUSED", fused_env)
    A = _complex_op(b2p_ctx, prob, terms, coefs)
    nd = prob.nd
    n = nd.ndofs
    Z = _elim(sum(c * M for c, M in zip(coefs, periodic["mats"])), nd.ess_dofs)
    Ki = periodic["mats"][2] + periodic["mats"][3]
    assert abs(Ki + Ki.T).max() < 1e-12 * abs(Ki).max()
    rng = np.random.default_rng(7)
    x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    yr, yi = torch.empty(n, dtype=torch.float64, device="cuda"), torch.empty(n, dtype=torch.float64, device="cuda")
    before = A.fused_applies()
    A.mult(_dev(x.real), _dev(x.imag), yr, yi)
    assert _rel(yr.cpu().numpy() + 1j * yi.cpu().numpy(), Z @ x) < RTOL
    A.mult_hermitian_transpose(_dev(x.real), _dev(x.imag), yr, yi)
    assert _rel(yr.cpu().numpy() + 1j * yi.cpu().numpy(), Z.conj().T @ x) < RTOL
    if fused_env == "1":
        assert A.fused_applies() == before + 2
    else:
        assert A.fused_applies() == before


def test_fgmres_with_complex_p_multigrid_on_the_periodic_box(b2p_ctx, periodic):
    """K - sigma M of the Floquet system (sigma < 0: Hermitian positive definite) by FGMRES preconditioned with a complex
    p-multigrid over orders {1, 2, 3}: Chebyshev smoothing, coarse levels p-coarsened from the fine operators (b2p_op_coarsen,
    fine quadrature), an accurate GMRES solve on the coarsest level."""
    from palace_b200 import capi

    capi.set_stream(b2p_ctx)
    prob, terms, coefs = periodic["prob"], periodic["terms"], periodic["coefs"]
    orders = [1, 2, 3]
    nd = {p: hs.build_nd_space(prob.mesh, prob.topo, p) for p in orders}
    A = {3: _complex_op(b2p_ctx, prob, terms, coefs)}
    for p in (2, 1):
        A[p] = _complex_op(b2p_ctx, prob, terms, coefs, space=nd[p], fine_ops=A[3].local_ops)
    P = [common.gpu_interp(b2p_ctx, nd[a], nd[b], asm.nd_prolongation_comps(a, b)) for a, b in zip(orders[:-1], orders[1:])]
    coarse = capi.ComplexSolver.krylov(b2p_ctx, 1, rel_tol=1e-13, max_it=1000, max_dim=1000)
    mg = capi.ComplexSolver.gmg(b2p_ctx, coarse, P, None, cycle_it=1, smooth_it=1, cheby_order=4)
    mg.gmg_set_operators([A[p] for p in orders])
    Ks = capi.ComplexSolver.krylov(b2p_ctx, capi.FGMRES, rel_tol=1e-10, max_it=200, max_dim=200)
    Ks.set_operator(A[3])
    Ks.set_preconditioner(mg)
    n = nd[3].ndofs
    rng = np.random.default_rng(31)
    b = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    b[nd[3].ess_dofs] = 0.0
    zr, zi = torch.zeros(n, dtype=torch.float64, device="cuda"), torch.zeros(n, dtype=torch.float64, device="cuda")
    Ks.mult(_dev(b.real), _dev(b.imag), zr, zi)
    st = Ks.stats()
    print("FGMRES + complex p-multigrid:", st)
    assert st["converged"] and st["its"] <= 110, st  # 95 in the CPU emulation of the same kernels
    Z = _elim(sum(c * M for c, M in zip(coefs, periodic["mats"])), nd[3].ess_dofs)
    assert _rel(zr.cpu().numpy() + 1j * zi.cpu().numpy(), spla.spsolve(Z.tocsc(), b)) < 1e-8


def test_mixed_kind_errors(b2p_ctx):
    from palace_b200 import capi

    prob = common.make_problem(n=(2, 2, 2), p=2, n_attr=2)
    geom = common.gpu_geom(b2p_ctx, prob)
    for kind in MIXED:
        with pytest.raises(capi.B2PError) as e:
            common.gpu_op(b2p_ctx, geom, prob, kind, mixed_ctx(kind, 2), assemble=True)
        assert "b2p error 3" in str(e.value) and "assembled q-data" in str(e.value)  # B2P_ERR_UNSUPPORTED
    # dense mixed terms still do not fuse
    n = prob.nd.ndofs
    ow, oc = dense_op(b2p_ctx, prob, O.ND_WEAKCURL, mixed_ctx(O.ND_WEAKCURL, 2)), dense_op(b2p_ctx, prob, O.ND_MIXEDCURL, mixed_ctx(O.ND_MIXEDCURL, 2))
    A = capi.Operator.par(b2p_ctx, n, n, [ow, oc], [0.7, 0.7], prob.nd.ess_dofs, diag_policy=1)
    assert not A.is_fused()


def test_dense_mixed_terms_in_a_complex_operator_hermitian_transpose(b2p_ctx, monkeypatch):
    """Dense-basis mixed terms applied term by term (they do not fuse): MultHermitianTranspose applies the transposed local
    operators, so it equals Z^H x also for the non-symmetric kinds."""
    from palace_b200 import capi

    prob = common.make_problem(n=(2, 2, 2), p=2, n_attr=2)
    n = prob.nd.ndofs
    terms = [(O.CURLCURL, common.coefficient(O.CURLCURL, 2)), (O.ND_MASS, common.coefficient(O.ND_MASS, 2)),
             (O.ND_WEAKCURL, mixed_ctx(O.ND_WEAKCURL, 2)), (O.ND_MIXEDCURL, mixed_ctx(O.ND_MIXEDCURL, 2, seed=8))]
    coefs = [1.0, -2.3 + 0.1j, 0.9j, 0.4 + 0.6j]
    Z = _elim(sum(c * common.oracle_matrix(prob, k, b, eliminate=False) for c, (k, b) in zip(coefs, terms)), prob.nd.ess_dofs)
    rng = np.random.default_rng(17)
    x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    for fused_env in ("1", "0"):
        monkeypatch.setenv("B2P_COMPLEX_FUSED", fused_env)
        ops = [dense_op(b2p_ctx, prob, k, b) for k, b in terms]
        A = capi.ComplexOperator.par(b2p_ctx, n, n, ops, coefs, prob.nd.ess_dofs, diag_policy=1)
        yr, yi = torch.empty(n, dtype=torch.float64, device="cuda"), torch.empty(n, dtype=torch.float64, device="cuda")
        A.mult(_dev(x.real), _dev(x.imag), yr, yi)
        assert _rel(yr.cpu().numpy() + 1j * yi.cpu().numpy(), Z @ x) < RTOL
        A.mult_hermitian_transpose(_dev(x.real), _dev(x.imag), yr, yi)
        assert _rel(yr.cpu().numpy() + 1j * yi.cpu().numpy(), Z.conj().T @ x) < RTOL


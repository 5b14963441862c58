"""GPU parity: the sm_90a sum-factorised kernels (through the C ABI) against the dense
reference-style CPU oracle on the same seeded inputs. Mirrors the structure of the reference's
"3D libCEED Operators" tests (/root/reference/test/unit/test-libceed.cpp:245-376,749-806): Mult,
diagonal; meshes with rotated element frames, curved (order-2) geometry, striped piecewise
matrix coefficients. FP64 tolerance: ||dy||_2 <= 1e-12 ||y||_2 (the reference's own bound is
||dy||^2 < 1e-12 max(||y||^2, 1), test-libceed.cpp:262-268; sum-factorisation only reorders sums)."""
import numpy as np
import pytest

from oracle import pyoracle as O
from tests import common

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

RTOL = 1e-12


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_geometry_qdata(b2p_ctx, p):
    prob = common.make_problem(p=p)
    g = common.gpu_geom(b2p_ctx, prob)
    qd = g.qdata()
    assert np.array_equal(qd[:, 0, :], prob.qdata_ref[:, 0, :])
    assert _rel(qd, prob.qdata_ref) < 1e-13
    g.close()


@pytest.mark.parametrize("assemble", [False, True])
@pytest.mark.parametrize("kind", [O.CURLCURL, O.ND_MASS, O.CURLCURL_MASS])
@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_nd_apply_matches_oracle(b2p_ctx, p, kind, assemble):
    prob = common.make_problem(p=p)
    blob = common.coefficient(kind, 3, "matrix", a_mass=1.3, a_curl=0.7)
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob, assemble)
    rng = np.random.default_rng(1)
    x = rng.random(prob.nd.ndofs)
    y_ref = common.oracle_apply(prob, kind, blob, x)
    xd, yd = _dev(x), torch.full((prob.nd.ndofs,), 7.0, dtype=torch.float64, device="cuda")
    op.apply(xd, yd)  # Mult: zero-fills
    torch.cuda.synchronize()
    assert _rel(yd.cpu().numpy(), y_ref) < RTOL
    op.apply_add(xd, yd)  # AddMult accumulates
    torch.cuda.synchronize()
    assert _rel(yd.cpu().numpy(), 2 * y_ref) < RTOL
    op.close()
    g.close()


@pytest.mark.parametrize("ctype", ["const", "scalar"])
def test_nd_apply_coefficient_types(b2p_ctx, ctype):
    prob = common.make_problem(p=3, warp=0.0, scramble=None, mesh_order=1)
    kind = O.CURLCURL_MASS
    blob = common.coefficient(kind, 3, ctype)
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob)
    x = np.random.default_rng(2).random(prob.nd.ndofs)
    yd = torch.empty(prob.nd.ndofs, dtype=torch.float64, device="cuda")
    op.apply(_dev(x), yd)
    assert _rel(yd.cpu().numpy(), common.oracle_apply(prob, kind, blob, x)) < RTOL


@pytest.mark.parametrize("p", [5, 6])
def test_nd_apply_high_order(b2p_ctx, p):
    prob = common.make_problem(n=(2, 1, 1), p=p, n_attr=2)
    kind = O.CURLCURL_MASS
    blob = common.coefficient(kind, 2, "matrix")
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob)
    x = np.random.default_rng(3).random(prob.nd.ndofs)
    yd = torch.empty(prob.nd.ndofs, dtype=torch.float64, device="cuda")
    op.apply(_dev(x), yd)
    assert _rel(yd.cpu().numpy(), common.oracle_apply(prob, kind, blob, x)) < RTOL


@pytest.mark.parametrize("assemble", [False, True])
@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_h1_diffusion_matches_oracle(b2p_ctx, p, assemble):
    prob = common.make_problem(p=p)
    blob = common.coefficient(O.H1_DIFFUSION, 3, "matrix")
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, O.H1_DIFFUSION, blob, assemble)
    x = np.random.default_rng(4).random(prob.h1.ndofs)
    yd = torch.empty(prob.h1.ndofs, dtype=torch.float64, device="cuda")
    op.apply(_dev(x), yd)
    assert _rel(yd.cpu().numpy(), common.oracle_apply(prob, O.H1_DIFFUSION, blob, x)) < RTOL


@pytest.mark.parametrize("assemble", [False, True])
@pytest.mark.parametrize("kind", [O.CURLCURL, O.ND_MASS, O.CURLCURL_MASS, O.H1_DIFFUSION])
@pytest.mark.parametrize("p", [1, 2, 3])
def test_diagonal_matches_oracle(b2p_ctx, p, kind, assemble):
    prob = common.make_problem(p=p)
    blob = common.coefficient(kind, 3, "matrix")
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob, assemble)
    d_ref = common.oracle_diag(prob, kind, blob)
    dd = torch.zeros(d_ref.size, dtype=torch.float64, device="cuda")
    op.diag_add(dd)
    assert _rel(dd.cpu().numpy(), d_ref) < RTOL


@pytest.mark.parametrize("pf,pc", [(2, 1), (3, 1), (3, 2), (4, 2)])
def test_coarsened_operator_shares_fine_quadrature(b2p_ctx, pf, pc):
    """CeedOperatorCoarsen semantics (libceed/operator.cpp:525-585): coarse-order basis, fine q-data."""
    from palace_b200.host import hexspace as hs

    prob = common.make_problem(p=pf)
    kind = O.CURLCURL_MASS
    blob = common.coefficient(kind, 3, "matrix")
    g = common.gpu_geom(b2p_ctx, prob)
    fine = common.gpu_op(b2p_ctx, g, prob, kind, blob)
    ndc = hs.build_nd_space(prob.mesh, prob.topo, pc)
    t = hs.tables_1d(pc, prob.q1d)
    idx, ori = ndc.native_restriction()
    coarse = fine.coarsen(pc, ndc.ndofs, idx, ori, ndc.dof_map, t.Bo, t.Bc, t.Gc)
    x = np.random.default_rng(5).random(ndc.ndofs)
    yd = torch.empty(ndc.ndofs, dtype=torch.float64, device="cuda")
    coarse.apply(_dev(x), yd)
    y_ref = common.oracle_apply(prob, kind, blob, x, space=ndc, q1d=prob.q1d)
    assert _rel(yd.cpu().numpy(), y_ref) < RTOL
    coarse.close()
    fine.close()


def test_prebuilt_qdata_path(b2p_ctx):
    from palace_b200 import capi

    prob = common.make_problem(p=2)
    g = capi.Geom.from_qdata(b2p_ctx, prob.qdata_ref, prob.q1d)
    kind = O.CURLCURL_MASS
    blob = common.coefficient(kind, 3, "matrix")
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob)
    x = np.random.default_rng(6).random(prob.nd.ndofs)
    yd = torch.empty(prob.nd.ndofs, dtype=torch.float64, device="cuda")
    op.apply(_dev(x), yd)
    assert _rel(yd.cpu().numpy(), common.oracle_apply(prob, kind, blob, x)) < RTOL


def test_set_coeff_updates_operator(b2p_ctx):
    prob = common.make_problem(p=2)
    kind = O.CURLCURL_MASS
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, common.coefficient(kind, 3, "const"), assemble=True)
    blob = common.coefficient(kind, 3, "matrix", a_mass=-2.0, a_curl=1.0)
    op.set_coeff(blob)
    x = np.random.default_rng(7).random(prob.nd.ndofs)
    yd = torch.empty(prob.nd.ndofs, dtype=torch.float64, device="cuda")
    op.apply(_dev(x), yd)
    assert _rel(yd.cpu().numpy(), common.oracle_apply(prob, kind, blob, x)) < RTOL


@pytest.mark.parametrize("kind", [O.CURLCURL, O.ND_MASS, O.CURLCURL_MASS])
@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_production_and_simple_kernels_agree_with_alpha_and_mask(b2p_ctx, p, kind):
    """b2p_op_apply_add_ex: alpha scaling, the essential-dof mask (ParOperator semantics,
    /root/reference/palace/linalg/rap.cpp:195-234) and the two kernel generations."""
    prob = common.make_problem(p=p)
    blob = common.coefficient(kind, 3, "matrix")
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob)
    ess = prob.nd.ess_dofs
    op.set_essential(ess)
    rng = np.random.default_rng(8)
    x = rng.random(prob.nd.ndofs)
    y0 = rng.random(prob.nd.ndofs)
    xm = x.copy()
    xm[ess] = 0.0
    y_ref = common.oracle_apply(prob, kind, blob, xm)
    y_ref[ess] = 0.0
    expect = y0 - 0.75 * y_ref
    for simple in (False, True):
        yd = _dev(y0)
        op.apply_add_ex(-0.75, _dev(x), yd, masked=True, simple_kernel=simple)
        torch.cuda.synchronize()
        assert _rel(yd.cpu().numpy(), expect) < RTOL


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_h1_production_and_simple_kernels_agree_with_alpha_and_mask(b2p_ctx, p):
    prob = common.make_problem(p=p)
    blob = common.coefficient(O.H1_DIFFUSION, 3, "matrix")
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, O.H1_DIFFUSION, blob)
    ess = prob.h1.ess_dofs
    op.set_essential(ess)
    rng = np.random.default_rng(12)
    x, y0 = rng.random(prob.h1.ndofs), rng.random(prob.h1.ndofs)
    xm = x.copy()
    xm[ess] = 0.0
    y_ref = common.oracle_apply(prob, O.H1_DIFFUSION, blob, xm)
    y_ref[ess] = 0.0
    for simple in (False, True):
        yd = _dev(y0)
        op.apply_add_ex(1.25, _dev(x), yd, masked=True, simple_kernel=simple)
        torch.cuda.synchronize()
        assert _rel(yd.cpu().numpy(), y0 + 1.25 * y_ref) < RTOL


@pytest.mark.parametrize("p", [2, 3])
@pytest.mark.parametrize("kind", [O.CURLCURL, O.ND_MASS, O.CURLCURL_MASS])
def test_both_production_nd_kernels_match_the_oracle(b2p_ctx, kind, p):
    """The default kernel -- nd_hex_apply7_kernel at p = 2 (one CTA per element batch, one 1-D line per thread), nd_hex_apply6_kernel
    at p = 3 (register x-gather, XDX on the Z region, aliased work arrays, half tables, branch-free scatter) -- and
    nd_hex_apply4_kernel, which B2P_APPLY_ROUND1_KERNEL selects for the same call. Both against the oracle: plain, scaled +
    masked, and over element sub-ranges with the owned | ghost split (a ragged last batch in each piece). The launch record says
    which kernel ran."""
    from palace_b200 import capi

    prob = common.make_problem(n=(3, 3, 2), p=p)
    blob = common.coefficient(kind, 3, "matrix", a_mass=0.9, a_curl=1.1)
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob)
    ess = prob.nd.ess_dofs
    op.set_essential(ess)
    rng = np.random.default_rng(23)
    x, y0 = rng.standard_normal(prob.nd.ndofs), rng.standard_normal(prob.nd.ndofs)
    y_ref = common.oracle_apply(prob, kind, blob, x)
    xm = x.copy()
    xm[ess] = 0.0
    ym = common.oracle_apply(prob, kind, blob, xm)
    ym[ess] = 0.0
    n_owned = prob.nd.ndofs // 2
    ne = prob.nd.lex_gid.shape[0]
    for r1 in (False, True):
        yd = _dev(y0)
        op.apply_add_ex(1.5, _dev(x), yd, round1_kernel=r1)
        assert _rel(yd.cpu().numpy(), y0 + 1.5 * y_ref) < RTOL
        assert capi.last_launch(b2p_ctx)["kernel"] == ("nd_hex_apply4_kernel" if r1 else {2: "nd_hex_apply7_kernel", 3: "nd_hex_apply6_kernel"}[p])
        yd = _dev(y0)
        op.apply_add_ex(-0.5, _dev(x), yd, masked=True, round1_kernel=r1)
        assert _rel(yd.cpu().numpy(), y0 - 0.5 * ym) < RTOL
        xd = _dev(x)
        yo = torch.zeros(n_owned, dtype=torch.float64, device="cuda")
        yg = torch.zeros(prob.nd.ndofs - n_owned, dtype=torch.float64, device="cuda")
        for e0, ec in ((0, ne // 3), (ne // 3, ne - ne // 3)):
            op.apply_add_split(1.0, xd[:n_owned].contiguous(), xd[n_owned:].contiguous(), yo, yg, n_owned, e0, ec, round1_kernel=r1)
        assert _rel(np.concatenate([yo.cpu().numpy(), yg.cpu().numpy()]), y_ref) < RTOL


@pytest.mark.parametrize("p", [4, 5, 6])
@pytest.mark.parametrize("kind", [O.CURLCURL, O.ND_MASS, O.CURLCURL_MASS])
def test_cta_per_batch_kernel_matches_the_oracle(b2p_ctx, kind, p):
    """nd_hex_apply7_kernel (p = 4, 5, 6: one CTA per element batch, warps specialised by vector component, one 1-D line per
    thread) against the oracle and against nd_hex_apply4_kernel on the same call: plain, scaled + masked, and over element
    sub-ranges with the owned | ghost split. 3 x 3 x 1 + 2 elements per piece leave a ragged last batch at p = 5 (two elements
    per batch)."""
    prob = common.make_problem(n=(3, 3, 1) if p == 6 else (3, 2, 2), p=p)
    blob = common.coefficient(kind, 3, "matrix", a_mass=0.9, a_curl=1.1)
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob)
    ess = prob.nd.ess_dofs
    op.set_essential(ess)
    rng = np.random.default_rng(29)
    x, y0 = rng.standard_normal(prob.nd.ndofs), rng.standard_normal(prob.nd.ndofs)
    y_ref = common.oracle_apply(prob, kind, blob, x)
    xm = x.copy()
    xm[ess] = 0.0
    ym = common.oracle_apply(prob, kind, blob, xm)
    ym[ess] = 0.0
    n_owned = prob.nd.ndofs // 2
    ne = prob.nd.lex_gid.shape[0]
    for cta in (True, False):
        yd = _dev(y0)
        op.apply_add_ex(1.5, _dev(x), yd, cta_kernel=cta, round1_kernel=not cta)
        assert _rel(yd.cpu().numpy(), y0 + 1.5 * y_ref) < RTOL
        yd = _dev(y0)
        op.apply_add_ex(-0.5, _dev(x), yd, masked=True, cta_kernel=cta, round1_kernel=not cta)
        assert _rel(yd.cpu().numpy(), y0 - 0.5 * ym) < RTOL
        xd = _dev(x)
        yo = torch.zeros(n_owned, dtype=torch.float64, device="cuda")
        yg = torch.zeros(prob.nd.ndofs - n_owned, dtype=torch.float64, device="cuda")
        for e0, ec in ((0, ne // 3 + 1), (ne // 3 + 1, ne - ne // 3 - 1)):
            op.apply_add_split(1.0, xd[:n_owned].contiguous(), xd[n_owned:].contiguous(), yo, yg, n_owned, e0, ec, cta_kernel=cta,
                               round1_kernel=not cta)
        assert _rel(np.concatenate([yo.cpu().numpy(), yg.cpu().numpy()]), y_ref) < RTOL


@pytest.mark.parametrize("p", [4, 5, 6])
def test_cta_per_batch_kernel_on_a_single_element_and_empty_ranges(b2p_ctx, p):
    """One element (a lone, partly filled batch at p = 5), an empty element range, and alpha = 0."""
    prob = common.make_problem(n=(1, 1, 1), p=p)
    kind = O.CURLCURL_MASS
    blob = common.coefficient(kind, 3, "matrix", a_mass=0.9, a_curl=1.1)
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob)
    rng = np.random.default_rng(37)
    n = prob.nd.ndofs
    x, y0 = rng.standard_normal(n), rng.standard_normal(n)
    y_ref = common.oracle_apply(prob, kind, blob, x)
    yd = _dev(y0)
    op.apply_add_ex(2.0, _dev(x), yd, cta_kernel=True)
    assert _rel(yd.cpu().numpy(), y0 + 2.0 * y_ref) < RTOL
    yd = _dev(y0)
    op.apply_add_ex(0.0, _dev(x), yd, cta_kernel=True)
    assert np.array_equal(yd.cpu().numpy(), y0)
    yo = torch.zeros(n, dtype=torch.float64, device="cuda")
    yg = torch.zeros(1, dtype=torch.float64, device="cuda")
    op.apply_add_split(1.0, _dev(x), yg, yo, yg, n, 1, 0, cta_kernel=True)  # no elements: nothing launched, nothing written
    assert not yo.cpu().numpy().any()


@pytest.mark.parametrize("p,cfgs", [(4, ["116d", "118g", "118c", "224g", "542c"]), (5, ["231d", "232g", "232c", "341g", "342c"]),
                                    (6, ["122g", "123d", "123c", "241c", "242g"])])
def test_cta_per_batch_kernel_launch_shapes(b2p_ctx, monkeypatch, p, cfgs):
    """The other launch shapes of nd_hex_apply7_kernel (B2P_ND7_CFG = elements per batch, warps per component, CTAs per SM,
    q-data by LDG (d), staged by TMA (g), staged by TMA with component-wide barriers (c)) compute the same operator: 14 elements leave ragged last batches for 3 and 5 elements
    per batch."""
    prob = common.make_problem(n=(7, 2, 1), p=p)
    kind = O.CURLCURL_MASS
    blob = common.coefficient(kind, 3, "matrix", a_mass=0.9, a_curl=1.1)
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob)
    rng = np.random.default_rng(31)
    x, y0 = rng.standard_normal(prob.nd.ndofs), rng.standard_normal(prob.nd.ndofs)
    y_ref = common.oracle_apply(prob, kind, blob, x)
    for cfg in cfgs:
        monkeypatch.setenv("B2P_ND7_CFG", cfg)
        yd = _dev(y0)
        op.apply_add_ex(0.75, _dev(x), yd, cta_kernel=True)
        assert _rel(yd.cpu().numpy(), y0 + 0.75 * y_ref) < RTOL, cfg


@pytest.mark.parametrize("assemble", [False, True])
@pytest.mark.parametrize("kind", [O.CURLCURL, O.ND_MASS, O.CURLCURL_MASS])
def test_halfwarp_kernel_matches_oracle(b2p_ctx, kind, assemble):
    """The one-element-per-warp p = 3 / q1d = 4 kernel (mirrored half-warps, b2p_hex_nd5.cu) against the oracle,
    with alpha and the essential-dof mask, on a warped mesh with scrambled element frames."""
    prob = common.make_problem(n=(3, 3, 2), p=3)
    blob = common.coefficient(kind, 3, "matrix", a_mass=0.9, a_curl=1.1)
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob, assemble)
    ess = prob.nd.ess_dofs
    op.set_essential(ess)
    rng = np.random.default_rng(21)
    x, y0 = rng.standard_normal(prob.nd.ndofs), rng.standard_normal(prob.nd.ndofs)
    y_ref = common.oracle_apply(prob, kind, blob, x)
    yd = _dev(y0)
    op.apply_add_ex(1.5, _dev(x), yd, halfwarp_kernel=True)
    torch.cuda.synchronize()
    assert _rel(yd.cpu().numpy(), y0 + 1.5 * y_ref) < RTOL
    xm = x.copy()
    xm[ess] = 0.0
    ym = common.oracle_apply(prob, kind, blob, xm)
    ym[ess] = 0.0
    yd = _dev(y0)
    op.apply_add_ex(-0.5, _dev(x), yd, masked=True, halfwarp_kernel=True)
    torch.cuda.synchronize()
    assert _rel(yd.cpu().numpy(), y0 - 0.5 * ym) < RTOL
    # owned / ghost split of the L-vector over an element sub-range, as the partitioned ParOperator calls it
    n_owned = prob.nd.ndofs // 2
    ne = prob.nd.lex_gid.shape[0]
    xd = _dev(x)
    for hw in (True, False):  # the default production kernel takes the same split path
        yo = torch.zeros(n_owned, dtype=torch.float64, device="cuda")
        yg = torch.zeros(prob.nd.ndofs - n_owned, dtype=torch.float64, device="cuda")
        for e0, ec in ((0, ne // 3), (ne // 3, ne - ne // 3)):
            op.apply_add_split(1.0, xd[:n_owned].contiguous(), xd[n_owned:].contiguous(), yo, yg, n_owned, e0, ec, halfwarp_kernel=hw)
        torch.cuda.synchronize()
        assert _rel(torch.cat([yo, yg]).cpu().numpy(), y_ref) < RTOL
    op.close()
    g.close()

"""nd_hex_apply7_kernel at p = 2 and 3 (one CTA per element batch, warps specialised by vector component, one 1-D line per
thread; the default at p = 2 for the symmetric kinds) against the oracle and against the round-1 kernel on the same call: the
three symmetric kinds and the block form of the two Floquet mixed curl kinds, alpha, the masked and transposed applies, the
owned | ghost split over element ranges with ragged last batches, one element, an empty range, alpha = 0, and every launch
shape of the B2P_ND7_CFG table at these orders."""
import numpy as np
import pytest

from oracle import pyoracle as O
from palace_b200.host import coeff as cf
from tests import common

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

RTOL = 1e-12
MIXED = [O.ND_WEAKCURL, O.ND_MIXEDCURL]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def _close(a, b, tol=1e-14):
    return np.abs(a - b).max() <= tol * np.abs(b).max()


def _blob(kind):
    if kind in MIXED:  # a non-symmetric matrix per material, as a Floquet wave vector gives
        am, mc = cf.test_suite_coefficient(3, "matrix")
        mc = mc + 0.3 * (np.random.default_rng(5).random(mc.shape) - 0.5)
        return cf.coeff_ctx(am, mc, a=-1.0) if kind == O.ND_WEAKCURL else cf.coeff_ctx(am, mc, a=1.0, transpose=True)
    return common.coefficient(kind, 3, "matrix", a_mass=0.9, a_curl=1.1)


@pytest.mark.parametrize("p", [2, 3])
@pytest.mark.parametrize("kind", [O.CURLCURL, O.ND_MASS, O.CURLCURL_MASS] + MIXED)
def test_cta_per_batch_kernel_matches_the_oracle_at_low_order(b2p_ctx, kind, p):
    """14 warped, scrambled elements; the split pieces of 5 and 9 elements end in partly filled batches at two (p = 3) and three
    (p = 2) elements per batch."""
    prob = common.make_problem(n=(7, 2, 1), p=p)
    blob = _blob(kind)
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob)
    ess = prob.nd.ess_dofs
    op.set_essential(ess)
    rng = np.random.default_rng(41 + p)
    n = prob.nd.ndofs
    x, y0 = rng.standard_normal(n), rng.standard_normal(n)
    y_ref = common.oracle_apply(prob, kind, blob, x)
    xm = x.copy()
    xm[ess] = 0.0
    ym = common.oracle_apply(prob, kind, blob, xm)
    ym[ess] = 0.0
    n_owned = n // 2
    ne = prob.nd.lex_gid.shape[0]
    out = {}
    for cta in (True, False):
        yd = _dev(y0)
        op.apply_add_ex(1.5, _dev(x), yd, cta_kernel=cta, round1_kernel=not cta)
        out["plain", cta] = yd.cpu().numpy()
        assert _rel(out["plain", cta], y0 + 1.5 * y_ref) < RTOL
        yd = _dev(y0)
        op.apply_add_ex(-0.5, _dev(x), yd, masked=True, cta_kernel=cta, round1_kernel=not cta)
        out["masked", cta] = yd.cpu().numpy()
        assert _rel(out["masked", cta], y0 - 0.5 * ym) < RTOL
        xd = _dev(x)
        yo = torch.zeros(n_owned, dtype=torch.float64, device="cuda")
        yg = torch.zeros(n - n_owned, dtype=torch.float64, device="cuda")
        for e0, ec in ((0, ne // 3 + 1), (ne // 3 + 1, ne - ne // 3 - 1)):
            op.apply_add_split(1.0, xd[:n_owned].contiguous(), xd[n_owned:].contiguous(), yo, yg, n_owned, e0, ec, cta_kernel=cta,
                               round1_kernel=not cta)
        out["split", cta] = np.concatenate([yo.cpu().numpy(), yg.cpu().numpy()])
        assert _rel(out["split", cta], y_ref) < RTOL
    for case in ("plain", "masked", "split"):  # the two kernels differ in the order of the sums only
        assert _close(out[case, True], out[case, False]), case
    # the default kernel (nd_hex_apply7_kernel at p = 2, nd_hex_apply6_kernel at p = 3 and for the block form) agrees with it
    yd = _dev(y0)
    op.apply_add_ex(1.5, _dev(x), yd)
    assert _close(yd.cpu().numpy(), out["plain", True])
    if kind in MIXED:
        A = common.oracle_matrix(prob, kind, blob, eliminate=False).tocsr()
        yd = _dev(y0)
        op.apply_add_ex(1.0, _dev(x), yd, transpose=True)
        assert _rel(yd.cpu().numpy(), y0 + A.T @ x) < RTOL


@pytest.mark.parametrize("kind", [O.CURLCURL_MASS, O.ND_MIXEDCURL])
@pytest.mark.parametrize("p", [2, 3])
def test_cta_per_batch_kernel_on_a_single_element_and_empty_ranges_at_low_order(b2p_ctx, p, kind):
    """One element (a lone, partly filled batch), an empty element range, and alpha = 0."""
    prob = common.make_problem(n=(1, 1, 1), p=p)
    blob = _blob(kind)
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob)
    rng = np.random.default_rng(43)
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


@pytest.mark.parametrize("p,cfgs", [(2, ["317c", "318d", "318g", "318c", "319c", "724g", "724c"]),
                                    (3, ["217c", "218d", "218g", "218c", "219c", "324c", "424g", "424c"])])
def test_cta_per_batch_kernel_launch_shapes_at_low_order(b2p_ctx, monkeypatch, p, cfgs):
    """The launch shapes of nd_hex_apply7_kernel at p = 2, 3 (B2P_ND7_CFG = elements per batch, warps per component, CTAs per
    SM, q-data by LDG (d), staged by TMA (g), staged by TMA with component-wide barriers (c)) compute the same operator: 14
    elements leave ragged last batches for 3 and 4 elements per batch."""
    prob = common.make_problem(n=(7, 2, 1), p=p)
    kind = O.CURLCURL_MASS
    blob = _blob(kind)
    g = common.gpu_geom(b2p_ctx, prob)
    op = common.gpu_op(b2p_ctx, g, prob, kind, blob)
    rng = np.random.default_rng(47)
    x, y0 = rng.standard_normal(prob.nd.ndofs), rng.standard_normal(prob.nd.ndofs)
    y_ref = common.oracle_apply(prob, kind, blob, x)
    for cfg in cfgs:
        monkeypatch.setenv("B2P_ND7_CFG", cfg)
        yd = _dev(y0)
        op.apply_add_ex(0.75, _dev(x), yd, cta_kernel=True)
        assert _rel(yd.cpu().numpy(), y0 + 0.75 * y_ref) < RTOL, cfg

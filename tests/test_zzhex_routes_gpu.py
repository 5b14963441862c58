"""Which element kernel each hexahedral apply runs (choose_hex_kernel in b2p_core.cu), pinned against the rules restated here.

For every order p = 1 ... 6 at q1d = p + 1 and p + 2, the three symmetric Nedelec kinds with stored and assembled q-data, a block
sum, the Raviart-Thomas mass and H1 diffusion, each apply flag: one apply on a tiny mesh, then the launch record
(capi.last_launch) names the kernel and its form, or -- for the cross-check kernels, which record nothing -- is unchanged.
B2P_ND_KERNEL is read once per process, so every forced value runs the same checks in a pytest subprocess of its own. The same
file pins the fused complex paths, the pair apply and the geometry bytes that depend on the route."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import pyoracle as O
from palace_b200.host import coeff as cf
from palace_b200.host import hexspace as hs
from tests import common

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

ND4, ND5, ND6, ND7, H1V3 = "nd_hex_apply4_kernel", "nd_hex_apply5_kernel", "nd_hex_apply6_kernel", "nd_hex_apply7_kernel", "h1_hex_apply3_kernel"
SYM = [O.CURLCURL, O.ND_MASS, O.CURLCURL_MASS]
FLAGS = ["simple_kernel", "halfwarp_kernel", "round1_kernel", "cta_kernel"]
PAIRS = [(p, q) for p in range(1, 7) for q in (p + 1, p + 2) if q <= 7]


def _forced():
    e = os.environ.get("B2P_ND_KERNEL")
    return int(e) if e else 0


def nd_route(p, q1d, assembled, flags, forced, block=False):
    """The Nedelec kernel of one apply (None: the cross-check kernel nd_hex_apply_kernel, which records nothing)."""
    simple, half, round1, cta = (f in flags for f in FLAGS)
    nd5 = p == 3 and q1d == 4
    nd6 = not assembled and q1d == p + 1 and p in (2, 3)
    nd7 = not assembled and q1d == p + 1 and 2 <= p <= 6
    if block:
        if simple or round1 or half or forced in (4, 5):
            return None
        if not (cta or forced == 7) and nd6:
            return ND6 + ":block"
        return ND7 + ":block" if nd7 else None
    if simple:
        return None
    if (half or forced == 5) and nd5:
        return ND5
    if (forced == 6 or (forced == 0 and p == 3)) and not (round1 or cta) and nd6:
        return ND6
    if (cta or forced in (0, 7)) and not round1 and nd7:
        return ND7
    return ND4


def _check(ctx, apply, kernel, what):
    from palace_b200 import capi

    try:
        seq = capi.last_launch(ctx)["seq"]
    except capi.B2PError:  # nothing recorded on this context yet
        seq = 0
    apply()
    torch.cuda.synchronize()
    r = capi.last_launch(ctx)
    if kernel is None:
        assert r["seq"] == seq, (what, r)
    else:
        assert r["seq"] > seq, (what, kernel)
        assert r["kernel"] == kernel, (what, r)


def _xy(n):
    return torch.from_numpy(np.random.default_rng(1).standard_normal(n)).cuda(), torch.zeros(n, dtype=torch.float64, device="cuda")


def test_routes(b2p_ctx):
    """Every case under this process's B2P_ND_KERNEL (unset: the default routes)."""
    from palace_b200 import capi
    from tests.test_zzhex_floquet_gpu import mixed_ctx

    forced = _forced()
    for p, q1d in PAIRS:
        prob = common.make_problem(n=(2, 1, 1), p=p, q1d=q1d)
        g = common.gpu_geom(b2p_ctx, prob)
        x, y = _xy(prob.nd.ndofs)
        for kind in SYM:
            blob = common.coefficient(kind, 3)
            for asm_ in (False, True):
                op = common.gpu_op(b2p_ctx, g, prob, kind, blob, asm_)
                sweep = [()] + [(f,) for f in FLAGS] if kind == O.CURLCURL_MASS else [(), ("simple_kernel",)]
                for flags in sweep:
                    _check(b2p_ctx, lambda: op.apply_add_ex(1.0, x, y, **{f: True for f in flags}), nd_route(p, q1d, asm_, flags, forced),
                           (p, q1d, kind, asm_, flags))
        terms = [common.gpu_op(b2p_ctx, g, prob, O.CURLCURL, common.coefficient(O.CURLCURL, 3)),
                 common.gpu_op(b2p_ctx, g, prob, O.ND_WEAKCURL, mixed_ctx(O.ND_WEAKCURL, 3))]
        S = capi.Op.create_sum(b2p_ctx, terms, [1.0, 0.5])
        for flags in [()] + [(f,) for f in FLAGS]:
            for tr in (False, True):
                _check(b2p_ctx, lambda: S.apply_add_ex(1.0, x, y, transpose=tr, **{f: True for f in flags}),
                       nd_route(p, q1d, False, flags, forced, block=True), (p, q1d, "block", flags, tr))
        h1 = common.gpu_op(b2p_ctx, g, prob, O.H1_DIFFUSION, common.coefficient(O.H1_DIFFUSION, 3))
        xh, yh = _xy(prob.h1.ndofs)
        _check(b2p_ctx, lambda: h1.apply_add_ex(1.0, xh, yh), H1V3, (p, q1d, "h1"))
        _check(b2p_ctx, lambda: h1.apply_add_ex(1.0, xh, yh, simple_kernel=True), None, (p, q1d, "h1 simple"))
        rt = hs.build_rt_space(prob.mesh, prob.topo, p)
        t = hs.tables_1d(p, q1d)
        R = capi.Op.create(b2p_ctx, g, capi.RT_MASS, p, rt.ndofs, rt.lex_gid, rt.lex_sign, None, t.Bo, t.Bc, None, cf.coeff_ctx(a=1.0))
        xr, yr = _xy(rt.ndofs)
        for flags in ((), ("simple_kernel",)):  # both Raviart-Thomas kernels record nothing
            _check(b2p_ctx, lambda: R.apply_add_ex(1.0, xr, yr, **{f: True for f in flags}), None, (p, q1d, "rt", flags))


def test_geometry_bytes_follow_the_route(b2p_ctx):
    """At p = 3 on a trilinear mesh the operator is charged the 8 vertices (192 bytes per element) exactly when it runs on
    nd_hex_apply6_kernel, which evaluates the geometry from them; every other route streams the q-data (80 bytes per point)."""
    forced = _forced()
    for p in (2, 3):
        prob = common.make_problem(n=(2, 1, 1), p=p, mesh_order=1)
        g = common.gpu_geom(b2p_ctx, prob)
        op = common.gpu_op(b2p_ctx, g, prob, O.CURLCURL_MASS, common.coefficient(O.CURLCURL_MASS, 3))
        geom = 192 if p == 3 and nd_route(p, p + 1, False, (), forced) == ND6 else 80 * prob.q1d ** 3
        ne, P = prob.mesh.ne, prob.nd.P
        assert op.algorithmic_bytes() == 16 * prob.nd.ndofs + ne * (4 * ((P + 3) & ~3) + geom + 144), (p, forced)


def _complex(ctx, prob, g, names):
    from palace_b200 import capi
    from tests.test_zzhex_floquet_gpu import mixed_ctx

    blobs = {"K": (O.CURLCURL, common.coefficient(O.CURLCURL, 3)), "M": (O.ND_MASS, common.coefficient(O.ND_MASS, 3)),
             "W": (O.ND_WEAKCURL, mixed_ctx(O.ND_WEAKCURL, 3))}
    ops = [common.gpu_op(ctx, g, prob, *blobs[n]) for n in names]
    A = capi.ComplexOperator.par(ctx, prob.nd.ndofs, prob.nd.ndofs, ops, [1.0, -2.0 + 0.1j, 0.5j][: len(ops)], prob.nd.ess_dofs, 1)
    A._keep = ops
    return A


@pytest.mark.parametrize("p", [1, 2, 3, 4])
def test_fused_complex_paths_and_pair_apply(b2p_ctx, p):
    """b2p_coperator_fused_path (2: nd_hex_apply4_kernel<CPLX>, 3: nd_hex_apply7_kernel<CPLX>, 1: two real sums, 0: term by term)
    and the kernel of the two-vector apply."""
    prob = common.make_problem(n=(2, 1, 1), p=p)
    g = common.gpu_geom(b2p_ctx, prob)
    assert _complex(b2p_ctx, prob, g, "KM").fused_path() == (2 if p <= 3 else 3)
    assert _complex(b2p_ctx, prob, g, "K").fused_path() == (2 if p <= 3 else 0)
    assert _complex(b2p_ctx, prob, g, "KMW").fused_path() == (3 if p >= 2 else 1)
    op = common.gpu_op(b2p_ctx, g, prob, O.CURLCURL_MASS, common.coefficient(O.CURLCURL_MASS, 3))
    x, y = _xy(prob.nd.ndofs)
    x1, y1 = _xy(prob.nd.ndofs)
    pair = ND4 + ":cplx" if p <= 3 else nd_route(p, p + 1, False, (), _forced())  # p >= 4: two real applies
    _check(b2p_ctx, lambda: op.apply_add_pair(1.0, x, x1, y, y1), pair, (p, "pair"))


@pytest.mark.skipif(os.environ.get("B2P_ND_KERNEL") is not None, reason="runs the forced values itself")
@pytest.mark.parametrize("forced", ["4", "5", "6", "7"])
def test_routes_under_forced_nd_kernel(forced):
    """B2P_ND_KERNEL = 4, 5, 6, 7: the checks above in a process of their own."""
    env = dict(os.environ, B2P_ND_KERNEL=forced)
    cmd = [sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider", __file__ + "::test_routes",
           __file__ + "::test_geometry_bytes_follow_the_route", __file__ + "::test_fused_complex_paths_and_pair_apply"]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]


def test_two_devices_in_one_process():
    """Kernel attributes (the dynamic shared memory allowance) belong to a device: contexts on devices 0 and 1 of one process
    each apply the p = 3 curl-curl + mass operator and match the oracle."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from palace_b200 import capi

    prob = common.make_problem(n=(3, 2, 2), p=3)
    kind = O.CURLCURL_MASS
    blob = common.coefficient(kind, 3)
    x = np.random.default_rng(0).random(prob.nd.ndofs)
    y_ref = common.oracle_apply(prob, kind, blob, x)
    keep = []
    for dev in (0, 1):
        with torch.cuda.device(dev):
            ctx = capi.Ctx(dev)
            op = common.gpu_op(ctx, common.gpu_geom(ctx, prob), prob, kind, blob)
            xd = torch.from_numpy(x).cuda()
            yd = torch.empty_like(xd)
            op.apply(xd, yd)
            torch.cuda.synchronize()
            keep += [ctx, op]
            assert np.linalg.norm(yd.cpu().numpy() - y_ref) <= 1e-12 * np.linalg.norm(y_ref), dev

"""Trilinear geometry evaluated inside nd_hex_apply6_kernel from the element vertices (b2p_geom_create_hex with mesh_order 1).

On an order-1 mesh the geometry object keeps the 8 vertices of every element, and the p = 2 / 3 Nedelec kernel evaluates w detJ and
adj(J)^T / detJ at each point from them instead of streaming the stored q-data. Both routes share one definition of the geometry
(b2p_geom1.cuh), so the same operator on Geom.from_qdata(geom.qdata()) -- the stored route in the same library -- must agree to
1e-14; both are checked against the oracle at 1e-12. The meshes are warped, scrambled boxes sized from the launch record so that
every warp walks several batches and the last batch is partly filled. The launch record says which geometry the kernel read."""
import math

import numpy as np
import pytest

from oracle import pyoracle as O
from tests import common
from tests.test_zzhex_floquet_gpu import mixed_ctx

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
RTOL, STORED_RTOL = 1e-12, 1e-14
ROUNDS = 2  # batches per warp at least
ND6, ND7 = "nd_hex_apply6_kernel", "nd_hex_apply7_kernel"
BLOCK_SUM = [(O.CURLCURL, 1.0), (O.ND_MASS, -2.0), (O.ND_WEAKCURL, 0.5)]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def _vec(n, seed):
    return np.random.default_rng(seed).standard_normal(n)


def _record(ctx):
    from palace_b200 import capi

    return capi.last_launch(ctx)


_PROBS = {}


def _problem(ctx, p):
    """Warped, scrambled order-1 box at order p: every warp of a full launch walks ROUNDS batches, the last one partly filled."""
    if p not in _PROBS:
        # a block operator runs on nd_hex_apply6_kernel at p = 2 and 3: its launch record gives the grid, warps and batch size
        tiny = common.make_problem(n=(2, 2, 2), p=p, mesh_order=1)
        op = common.gpu_op(ctx, common.gpu_geom(ctx, tiny), tiny, O.ND_WEAKCURL, mixed_ctx(O.ND_WEAKCURL, 3))
        n = tiny.nd.ndofs
        op.apply(_dev(_vec(n, 1)), torch.zeros(n, dtype=torch.float64, device="cuda"))
        r = _record(ctx)
        assert r["kernel"] == ND6 + ":block", r
        epb = r["elems_per_batch"]
        k = max(3, math.ceil((ROUNDS * r["max_grid"] * r["workers"] * epb + 1) ** (1.0 / 3.0))) | 1
        dims = [k, k, k]  # odd sizes: never a multiple of 2 elements, and of 3 only until nx grows by 2
        while (dims[0] * dims[1] * dims[2]) % epb == 0:
            dims[0] += 2
        _PROBS[p] = common.make_problem(n=tuple(dims), p=p, mesh_order=1)
    return _PROBS[p]


def _geoms(ctx, prob):
    """Node geometry of the mesh and the same geometry as stored q-data."""
    from palace_b200 import capi

    g = common.gpu_geom(ctx, prob)
    return g, capi.Geom.from_qdata(ctx, g.qdata(), prob.q1d)


def _ran(ctx, kernel, geom):
    """The last persistent launch was `kernel` (name and form) reading the geometry from `geom` ("nodes" or "qdata")."""
    r = _record(ctx)
    assert (r["kernel"], r["geom"]) == (kernel, geom), r
    return r


COEFFS = {"iso": dict(coeff_type="const", a_mass=0.7, a_curl=1.3), "matrix": dict(coeff_type="matrix")}


@pytest.mark.parametrize("coeff", ["iso", "matrix"])
@pytest.mark.parametrize("kind", [O.CURLCURL, O.ND_MASS, O.CURLCURL_MASS], ids=["curlcurl", "mass", "curlcurl_mass"])
@pytest.mark.parametrize("p", [2, 3])
def test_symmetric_kinds(b2p_ctx, p, kind, coeff):
    """Default apply, alpha, the essential-dof mask and the owned | ghost split over two element ranges (the boundary inside a
    batch): node geometry against the oracle and against the stored route. At p = 2 the symmetric kinds run on
    nd_hex_apply7_kernel, which reads the stored q-data of the same geometry object."""
    prob = _problem(b2p_ctx, p)
    nd, ne = prob.nd, prob.mesh.ne
    n, ess = nd.ndofs, nd.ess_dofs
    blob = common.coefficient(kind, 3, **COEFFS[coeff])
    g_nodes, g_stored = _geoms(b2p_ctx, prob)
    ops = {"nodes": common.gpu_op(b2p_ctx, g_nodes, prob, kind, blob), "qdata": common.gpu_op(b2p_ctx, g_stored, prob, kind, blob)}
    kernel, geom = (ND6, "nodes") if p == 3 else (ND7, "qdata")
    x, y0 = _vec(n, 1), _vec(n, 7)
    xm = x.copy()
    xm[ess] = 0.0
    y_ref = common.oracle_apply(prob, kind, blob, x)
    ym = common.oracle_apply(prob, kind, blob, xm)
    ym[ess] = 0.0
    xd = _dev(x)
    out = {}
    for route, op in ops.items():
        op.set_essential(ess)
        res = []
        y = torch.full((n,), float("nan"), dtype=torch.float64, device="cuda")
        op.apply(xd, y)
        res.append(y.cpu().numpy())
        yd = _dev(y0)
        op.apply_add_ex(1.5, xd, yd)
        res.append((yd.cpu().numpy() - y0) / 1.5)
        yd = _dev(y0)
        op.apply_add_ex(-0.75, xd, yd, masked=True)
        res.append((yd.cpu().numpy() - y0) / -0.75)
        r = _ran(b2p_ctx, kernel, geom if route == "nodes" else "qdata")
        if kernel == ND6:
            assert r["batches"] >= ROUNDS * r["grid"] * r["workers"] and ne % r["elems_per_batch"] != 0, r
        n_owned, epb = n // 2, r["elems_per_batch"]
        e1 = epb * (ne // (3 * epb)) + 1
        yo = torch.zeros(n_owned, dtype=torch.float64, device="cuda")
        yg = torch.zeros(n - n_owned, dtype=torch.float64, device="cuda")
        for e0, ec in ((0, e1), (e1, ne - e1)):
            op.apply_add_split(1.0, xd[:n_owned].contiguous(), xd[n_owned:].contiguous(), yo, yg, n_owned, e0, ec)
        _ran(b2p_ctx, kernel, geom if route == "nodes" else "qdata")
        res.append(np.concatenate([yo.cpu().numpy(), yg.cpu().numpy()]))
        for got, ref in zip(res, [y_ref, y_ref, ym, y_ref]):
            assert _rel(got, ref) < RTOL, route
        out[route] = res
    for a, b in zip(out["nodes"], out["qdata"]):
        assert _rel(a, b) < STORED_RTOL


@pytest.mark.parametrize("which", ["W", "X", "S"], ids=["weakcurl", "mixedcurl", "curlcurl_mass_weakcurl"])
@pytest.mark.parametrize("p", [2, 3])
def test_block_forms(b2p_ctx, p, which):
    """The block operators (mixed curl kinds and a fused sum with one) forward and transposed on a trilinear geometry: they keep
    the stored q-data (their kernel has no registers left for the vertex route), against the oracle (transposed: by the adjoint
    identity) and against the same operators on the q-data alone, with the same byte count."""
    from palace_b200 import capi

    prob = _problem(b2p_ctx, p)
    n = prob.nd.ndofs
    x, u = _vec(n, 1), _vec(n, 5)
    blobs = {"K": common.coefficient(O.CURLCURL, 3), "M": common.coefficient(O.ND_MASS, 3), "W": mixed_ctx(O.ND_WEAKCURL, 3),
             "X": mixed_ctx(O.ND_MIXEDCURL, 3)}
    kinds = {"K": O.CURLCURL, "M": O.ND_MASS, "W": O.ND_WEAKCURL, "X": O.ND_MIXEDCURL}
    if which == "S":
        names = {O.CURLCURL: "K", O.ND_MASS: "M", O.ND_WEAKCURL: "W"}
        y_ref = sum(c * common.oracle_apply(prob, k, blobs[names[k]], x) for k, c in BLOCK_SUM)
    else:
        y_ref = common.oracle_apply(prob, kinds[which], blobs[which], x)

    def make(geom):
        if which != "S":
            return common.gpu_op(b2p_ctx, geom, prob, kinds[which], blobs[which])
        terms = [common.gpu_op(b2p_ctx, geom, prob, kinds[k], blobs[k]) for k in ("K", "M", "W")]
        S = capi.Op.create_sum(b2p_ctx, terms, [c for _, c in BLOCK_SUM])
        S._keep = terms
        return S

    g_nodes, g_stored = _geoms(b2p_ctx, prob)
    out, nbytes = {}, {}
    for route, geom in (("nodes", g_nodes), ("qdata", g_stored)):
        op = make(geom)
        nbytes[route] = op.algorithmic_bytes()
        y = torch.full((n,), float("nan"), dtype=torch.float64, device="cuda")
        op.apply(_dev(x), y)
        _ran(b2p_ctx, ND6 + ":block", "qdata")
        yt = torch.zeros(n, dtype=torch.float64, device="cuda")
        op.apply_add_ex(1.0, _dev(u), yt, transpose=True)
        _ran(b2p_ctx, ND6 + ":block", "qdata")
        y, yt = y.cpu().numpy(), yt.cpu().numpy()
        assert _rel(y, y_ref) < RTOL, route
        assert abs(x @ yt - y_ref @ u) <= RTOL * np.linalg.norm(y_ref) * np.linalg.norm(u), route
        out[route] = (y, yt)
    for a, b in zip(out["nodes"], out["qdata"]):
        assert _rel(a, b) < STORED_RTOL
    assert nbytes["nodes"] == nbytes["qdata"]


def test_stored_qdata_and_bytes_of_node_geometry(b2p_ctx):
    """The q-data of an order-1 geometry (still stored for the other kernels) equals the oracle's. The byte count of an operator
    that reads the vertices charges 192 bytes of geometry per element instead of 80 per point; operators whose kernel streams the
    q-data of the same geometry (the symmetric kinds at p = 2 on nd_hex_apply7_kernel, the Raviart-Thomas mass) are charged the
    q-data."""
    from palace_b200 import capi
    from palace_b200.host import coeff as cf
    from palace_b200.host import hexspace as hs

    prob = _problem(b2p_ctx, 3)
    g_nodes, g_stored = _geoms(b2p_ctx, prob)
    qd = g_nodes.qdata()
    assert np.array_equal(qd[:, 0], prob.qdata_ref[:, 0])  # attributes
    assert np.abs(qd[:, 1:] - prob.qdata_ref[:, 1:]).max() <= 1e-13 * np.abs(prob.qdata_ref[:, 1:]).max()
    blob = common.coefficient(O.CURLCURL_MASS, 3)
    a = common.gpu_op(b2p_ctx, g_nodes, prob, O.CURLCURL_MASS, blob).algorithmic_bytes()
    b = common.gpu_op(b2p_ctx, g_stored, prob, O.CURLCURL_MASS, blob).algorithmic_bytes()
    assert b - a == prob.mesh.ne * (80 * prob.q1d ** 3 - 192)
    prob2 = _problem(b2p_ctx, 2)
    g2_nodes, g2_stored = _geoms(b2p_ctx, prob2)
    a2 = common.gpu_op(b2p_ctx, g2_nodes, prob2, O.CURLCURL_MASS, blob).algorithmic_bytes()
    assert a2 == common.gpu_op(b2p_ctx, g2_stored, prob2, O.CURLCURL_MASS, blob).algorithmic_bytes()
    rt = hs.build_rt_space(prob.mesh, prob.topo, 3)
    t = hs.tables_1d(3, prob.q1d)

    def rt_bytes(geom):
        op = capi.Op.create(b2p_ctx, geom, capi.RT_MASS, 3, rt.ndofs, rt.lex_gid, rt.lex_sign, None, t.Bo, t.Bc, None, cf.coeff_ctx(a=1.0))
        return op.algorithmic_bytes()

    assert rt_bytes(g_nodes) == rt_bytes(g_stored)

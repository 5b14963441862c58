"""The persistent element kernels in their steady state, against the oracle.

nd_hex_apply4/5/6/7_kernel and h1_hex_apply3_kernel clamp their grid to the element batches and let every worker (a warp, or the
whole CTA for nd_hex_apply7_kernel) walk batch, batch + W, ... over the W workers of the grid. Part of their code runs only from
a worker's second batch onward: the wait on the next ring slot and the gather of the next batch's x, the refill of the q-data
buffers, the reissue of a ring slot three batches ahead, every flip of an mbarrier phase parity. Small meshes give each worker
one batch at most, so none of that runs there.

Every case here sizes its mesh from the launch record of the library (capi.last_launch): one apply on a tiny mesh gives the
CTAs per launch before clamping, the workers per CTA and the elements per batch; the warped, scrambled box then grows until
every worker walks at least ROUNDS batches, with a partly filled last batch and an uneven last wave. After each apply the record
says which kernel ran and that it ran in that steady state. The same file is therefore small on the emulated machine
(tests/test_emulated_kernels.py, one emulated SM) and full-sized on the GPU.

Every result is checked against the oracle at 1e-12 relative (FP64, different summation order)."""
import functools
import math

import numpy as np
import pytest

from oracle import pyoracle as O
from palace_b200.host import coeff as cf
from palace_b200.host import hexmesh as hm
from palace_b200.host import hexspace as hs
from tests import common
from tests.test_cylinder_floquet_golden import cross_matrix
from tests.test_zzhex_floquet_gpu import mixed_ctx

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
RTOL = 1e-12
ROUNDS = 4  # batches per worker at least: every ring slot is reused and every mbarrier parity flips

ND4, ND5, ND6, ND7, H1V3 = "nd_hex_apply4_kernel", "nd_hex_apply5_kernel", "nd_hex_apply6_kernel", "nd_hex_apply7_kernel", "h1_hex_apply3_kernel"
SYM = [O.CURLCURL, O.ND_MASS, O.CURLCURL_MASS]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _nan(n):
    return torch.full((n,), float("nan"), dtype=torch.float64, device="cuda")


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


# ------------------------------------------------------------------------------------------------------------ launch records
_last_seq = [0]


def _record(ctx):
    from palace_b200 import capi

    return capi.last_launch(ctx)


def _ran(ctx, kernel, ne=None):
    """The apply just made launched `kernel` (name and form) and every worker walked at least ROUNDS batches; with `ne` (a
    launch over all ne elements) also a partly filled last batch and an uneven last wave."""
    r = _record(ctx)
    assert r["seq"] > _last_seq[0], f"no persistent launch recorded (expected {kernel})"
    _last_seq[0] = r["seq"]
    assert r["kernel"] == kernel, r
    assert r["grid"] == r["max_grid"], r
    assert r["batches"] >= ROUNDS * r["grid"] * r["workers"], r
    if ne is not None:
        assert r["batches"] == -(-ne // r["elems_per_batch"]), r
        assert r["elems_per_batch"] == 1 or ne % r["elems_per_batch"] != 0, r
        assert r["grid"] * r["workers"] == 1 or r["batches"] % (r["grid"] * r["workers"]) != 0, r
    return r


def _probe(ctx, launch):
    """Launch record of one apply on a tiny mesh."""
    launch()
    torch.cuda.synchronize()
    r = _record(ctx)
    _last_seq[0] = r["seq"]
    return r


def _fits(ne, r):
    W, epb = r["max_grid"] * r["workers"], r["elems_per_batch"]
    nb = -(-ne // epb)
    # the larger piece of the owned | ghost split (7/8 of the elements) still walks ROUNDS batches per worker
    big = -(-(ne - ne // 8 - 1) // epb)
    return big >= ROUNDS * W and (W == 1 or nb % W != 0) and (epb == 1 or ne % epb != 0)


def _box(records, min_nz=2):
    """The smallest near-cubic box whose element count fits every launch record."""
    need = max(math.ceil((ROUNDS * r["max_grid"] * r["workers"] * r["elems_per_batch"] + 1) * 8 / 7) for r in records)
    c = need ** (1.0 / 3.0)
    best = None
    for nz in range(max(min_nz, int(c / 2)), int(2 * c) + 3):
        for ny in range(max(2, int(c / 2)), int(2 * c) + 3):
            nx0 = max(2, -(-need // (ny * nz)))
            for nx in range(nx0, nx0 + 16):
                ne = nx * ny * nz
                if best is not None and ne >= best[0]:
                    break
                if all(_fits(ne, r) for r in records):
                    best = (ne, (nx, ny, nz))
                    break
    assert best is not None, records
    return best[1]


# ------------------------------------------------------------------------------------------------------------ problems
BLOBS = {
    "K": (O.CURLCURL, dict(coeff_type="matrix")),
    "M": (O.ND_MASS, dict(coeff_type="matrix")),
    "KM": (O.CURLCURL_MASS, dict(coeff_type="matrix")),
    "C": (O.ND_MASS, dict(coeff_type="scalar", a_mass=0.3)),
}
SYM_NAME = {O.CURLCURL: "K", O.ND_MASS: "M", O.CURLCURL_MASS: "KM"}
CPLX_SUM = [("K", 1.0 + 0.0j), ("M", -4.0 * (1 - 0.02j)), ("C", 2.0j)]  # K - w^2 (1 - i tan d) M + i w C
BLOCK_SUM = [(O.CURLCURL, 1.0), (O.ND_MASS, -2.0), (O.ND_WEAKCURL, 0.5)]  # curl-curl + mass + weak curl, one block operator


def _blob(name):
    if name in BLOBS:
        kind, kw = BLOBS[name]
        return kind, common.coefficient(kind, 3, **kw)
    kind = {"W": O.ND_WEAKCURL, "X": O.ND_MIXEDCURL}[name]
    return kind, mixed_ctx(kind, 3)


def _floquet_terms():
    """The five terms of a Floquet system on a z-periodic box: curl-curl, the k-mass, i (weak curl + mixed curl), a mass shift."""
    kx = cross_matrix((0.0, 0.0, 0.4))
    am = np.array([0])
    terms = [(O.CURLCURL, cf.coeff_ctx(a=1.0)), (O.ND_MASS, cf.coeff_ctx(am, (kx.T @ kx)[None])),
             (O.ND_WEAKCURL, cf.coeff_ctx(am, kx[None], a=-1.0)), (O.ND_MIXEDCURL, cf.coeff_ctx(am, kx[None], transpose=True)),
             (O.ND_MASS, cf.coeff_ctx(a=1.0))]
    return terms, [1.0, 1.0, 1j, 1j, 1.5]


def _tiny(p, q1d=None, periodic=False):
    if periodic:
        return common.problem_on_mesh(hm.box_mesh((2, 1, 3), (1.0, 0.8, 0.9), warp_amp=0.04, scramble_seed=11, periodic_z=True), p, q1d)
    return common.make_problem(n=(2, 2, 2), p=p, q1d=q1d)


_PROBS = {}


def _problem(key, n, p, q1d=None, periodic=False):
    if key not in _PROBS:
        if periodic:
            mesh = hm.box_mesh(n, (1.0, 0.8, 0.9), warp_amp=0.04, scramble_seed=11, periodic_z=True)
            _PROBS[key] = common.problem_on_mesh(mesh, p, q1d)
        else:
            _PROBS[key] = common.make_problem(n=n, p=p, q1d=q1d)
    return _PROBS[key]


def _vector(n, name):
    return np.random.default_rng({"x": 1, "xi": 3, "u": 5, "y0": 7}[name]).standard_normal(n)


def _masked(prob, name):
    v = _vector(prob.nd.ndofs, name)
    v[prob.nd.ess_dofs] = 0.0
    return v


@functools.lru_cache(maxsize=None)
def _oracle(key, name, vec, masked=False):
    """Oracle apply of the term `name` on the problem `key` to a named vector (optionally with the essential entries zeroed)."""
    if name == "KM":  # the pair context holds the contexts of "M" and "K": the sum of their applies
        return _oracle(key, "K", vec, masked) + _oracle(key, "M", vec, masked)
    prob = _PROBS[key]
    kind, blob = _blob(name)
    v = _masked(prob, vec) if masked else _vector(prob.nd.ndofs, vec)
    return common.oracle_apply(prob, kind, blob, v)


def _op(ctx, prob, name, assemble=False, geom=None):
    kind, blob = _blob(name)
    geom = common.gpu_geom(ctx, prob) if geom is None else geom
    return common.gpu_op(ctx, geom, prob, kind, blob, assemble)


def _block_ops(ctx, prob):
    """The two mixed kinds and the fused curl-curl + mass + weak-curl sum: block operators."""
    from palace_b200 import capi

    g = common.gpu_geom(ctx, prob)
    W, X = _op(ctx, prob, "W", geom=g), _op(ctx, prob, "X", geom=g)
    terms = [_op(ctx, prob, n_, geom=g) for n_ in ("K", "M")] + [W]
    S = capi.Op.create_sum(ctx, terms, [c for _, c in BLOCK_SUM])
    S._keep = terms
    return {"W": W, "X": X, "S": S}


def _complex_sum(ctx, prob, geom=None):
    from palace_b200 import capi

    g = common.gpu_geom(ctx, prob) if geom is None else geom
    ops = [_op(ctx, prob, n_, geom=g) for n_, _ in CPLX_SUM]
    return capi.ComplexOperator.par(ctx, prob.nd.ndofs, prob.nd.ndofs, ops, [c for _, c in CPLX_SUM], prob.nd.ess_dofs, 1)


def _par(ctx, prob, name):
    from palace_b200 import capi

    op = _op(ctx, prob, name)
    A = capi.Operator.par(ctx, prob.nd.ndofs, prob.nd.ndofs, [op], None, prob.nd.ess_dofs, diag_policy=1)
    A._keep.append(op)
    return A


# ------------------------------------------------------------------------------------------------------------ routes per order
def _real_routes(p):
    """(label, apply flags, assembled q-data, kernel) of the real symmetric kinds at q1d = p + 1."""
    default = {1: ND4, 2: ND7, 3: ND6}.get(p, ND7)
    routes = [("default", {}, False, default)]
    if p >= 2:
        routes.append(("round1", {"round1_kernel": True}, False, ND4))
    if p == 3:
        routes += [("halfwarp", {"halfwarp_kernel": True}, False, ND5), ("cta", {"cta_kernel": True}, False, ND7)]
    routes.append(("assembled", {}, True, ND4))
    return routes


def _block_kernel(p):
    return (ND6 if p <= 3 else ND7) + ":block"


def _complex_kernel(p):
    return (ND4 if p <= 3 else ND7) + ":cplx"


def _probes(ctx, p):
    """Launch records of every case on the non-periodic box at order p."""
    prob = _tiny(p)
    n = prob.nd.ndofs
    x, y = _dev(_vector(n, "x")), torch.zeros(n, dtype=torch.float64, device="cuda")
    g = common.gpu_geom(ctx, prob)
    recs = []
    for kind in SYM:
        for _, flags, asm_, _ in _real_routes(p):
            op = _op(ctx, prob, SYM_NAME[kind], asm_, geom=g)
            recs.append(_probe(ctx, lambda: op.apply_add_ex(1.0, x, y, **flags)))
    A = _complex_sum(ctx, prob, g)
    yi = torch.zeros_like(y)
    recs.append(_probe(ctx, lambda: A.mult(x, x, y, yi)))
    if p >= 2:
        for B in _block_ops(ctx, prob).values():
            recs.append(_probe(ctx, lambda: B.apply(x, y)))
    if p in PDL_ORDERS:
        P = _par(ctx, prob, "KM")
        recs.append(_probe(ctx, lambda: P.mult(x, y)))
    return recs


PDL_ORDERS = (3, 5)
_BOXES = {}


def _steady_problem(ctx, p):
    """The non-periodic box at order p (q1d = p + 1) sized for every case of this file at that order."""
    if p not in _BOXES:
        _BOXES[p] = _box(_probes(ctx, p))
    return ("sym", p), _problem(("sym", p), _BOXES[p], p)


# ------------------------------------------------------------------------------------------------------------ 1. real symmetric kinds
def _check_real(ctx, key, prob, name, op, routes):
    """apply into NaN (default route), apply_add_ex with alpha and with alpha + the essential-dof mask, and the owned | ghost
    split over two element ranges whose boundary falls inside a batch -- on every route."""
    nd = prob.nd
    n, ne, ess = nd.ndofs, prob.mesh.ne, nd.ess_dofs
    op.set_essential(ess)
    x, y0 = _vector(n, "x"), _vector(n, "y0")
    y_ref = _oracle(key, name, "x")
    ym = _oracle(key, name, "x", masked=True).copy()
    ym[ess] = 0.0
    n_owned = n // 2
    xd = _dev(x)
    for label, flags, _, kernel in routes:
        if label in ("default", "assembled"):
            y = _nan(n)
            op.apply(xd, y)
            assert _rel(y.cpu().numpy(), y_ref) < RTOL, label
            r = _ran(ctx, kernel, ne)
        yd = _dev(y0)
        op.apply_add_ex(1.5, xd, yd, **flags)
        assert _rel(yd.cpu().numpy(), y0 + 1.5 * y_ref) < RTOL, label
        r = _ran(ctx, kernel, ne)
        yd = _dev(y0)
        op.apply_add_ex(-0.75, xd, yd, masked=True, **flags)
        assert _rel(yd.cpu().numpy(), y0 - 0.75 * ym) < RTOL, label
        _ran(ctx, kernel, ne)
        epb = r["elems_per_batch"]
        e1 = ne // 8 if epb == 1 else epb * (ne // (8 * epb)) + 1  # inside a batch of the whole-range launch
        yo = torch.zeros(n_owned, dtype=torch.float64, device="cuda")
        yg = torch.zeros(n - n_owned, dtype=torch.float64, device="cuda")
        for e0, ec in ((0, e1), (e1, ne - e1)):
            op.apply_add_split(1.0, xd[:n_owned].contiguous(), xd[n_owned:].contiguous(), yo, yg, n_owned, e0, ec, **flags)
        _ran(ctx, kernel)
        assert _rel(np.concatenate([yo.cpu().numpy(), yg.cpu().numpy()]), y_ref) < RTOL, label


@pytest.mark.parametrize("kind", SYM, ids=["curlcurl", "mass", "curlcurl_mass"])
@pytest.mark.parametrize("p", [1, 2, 3, 4, 5, 6])
def test_real_symmetric_kinds(b2p_ctx, p, kind):
    key, prob = _steady_problem(b2p_ctx, p)
    name = SYM_NAME[kind]
    g = common.gpu_geom(b2p_ctx, prob)
    routes = _real_routes(p)
    _check_real(b2p_ctx, key, prob, name, _op(b2p_ctx, prob, name, geom=g), [r for r in routes if not r[2]])
    _check_real(b2p_ctx, key, prob, name, _op(b2p_ctx, prob, name, assemble=True, geom=g), [r for r in routes if r[2]])


# coarsened operators that keep the fine quadrature: the auxiliary levels of a p-multigrid (nd_hex_apply4_kernel at q1d > p + 1)
@pytest.mark.parametrize("kind", SYM, ids=["curlcurl", "mass", "curlcurl_mass"])
@pytest.mark.parametrize("p,q1d", [(1, 4), (2, 5), (1, 7)])
def test_coarsened_operators_keep_the_fine_quadrature(b2p_ctx, p, q1d, kind):
    name = SYM_NAME[kind]

    def coarse_op(prob):
        fine_nd = hs.build_nd_space(prob.mesh, prob.topo, q1d - 1)  # the fine level: order q1d - 1 at its default quadrature
        fine = common.gpu_op(b2p_ctx, common.gpu_geom(b2p_ctx, prob), prob, *_blob(name), space=fine_nd)
        t = hs.tables_1d(p, q1d)
        idx, ori = prob.nd.native_restriction()
        op = fine.coarsen(p, prob.nd.ndofs, idx, ori, prob.nd.dof_map, t.Bo, t.Bc, t.Gc)
        op._fine = fine
        return op

    tiny = _tiny(p, q1d)
    n = tiny.nd.ndofs
    op = coarse_op(tiny)
    rec = _probe(b2p_ctx, lambda: op.apply_add_ex(1.0, _dev(_vector(n, "x")), torch.zeros(n, dtype=torch.float64, device="cuda")))
    key = ("coarse", p, q1d, name)
    prob = _problem(key, _box([rec]), p, q1d)
    _check_real(b2p_ctx, key, prob, name, coarse_op(prob), [("default", {}, False, ND4)])


# ------------------------------------------------------------------------------------------------------------ 2. H1 diffusion
H1_PAIRS = [(p, q) for p in range(1, 7) for q in range(p + 1, 8)]


def _h1_problem(n, p, q1d):
    """Spaces, tables and oracle q-data of an H1 problem (no Nedelec space)."""
    mesh = hm.box_mesh(n, (1.0, 0.7, 0.9), warp_amp=0.04, scramble_seed=3, n_attr=3)
    topo = hs.build_topology(mesh)
    nodes = hs.gauss_lobatto(3)
    qx, _ = hs.gauss_legendre(q1d)
    nB, nG = hs.lagrange_table(nodes, qx)
    qd = O.geom_hex_qdata(mesh.node_coords(2, nodes), mesh.attr, 2, q1d)
    return common.Problem(mesh, topo, p, q1d, 2, mesh.node_coords(2, nodes), None, hs.build_h1_space(mesh, topo, p), hs.tables_1d(p, q1d),
                          (nB, nG), qd)


_H1 = {}


def _h1_case(ctx, p, q1d):
    """The H1 box at (p, q1d) sized for stored and assembled q-data, its oracle applies to x and to x with the essential entries
    zeroed (one problem at a time: the stored and the assembled case follow each other)."""
    blob = common.coefficient(O.H1_DIFFUSION, 3, "matrix")
    if (p, q1d) not in _H1:
        _H1.clear()
        tiny = _h1_problem((2, 2, 2), p, q1d)
        g = common.gpu_geom(ctx, tiny)
        n = tiny.h1.ndofs
        x, y = _dev(_vector(n, "x")), torch.zeros(n, dtype=torch.float64, device="cuda")
        recs = []
        for assemble in (False, True):
            op = common.gpu_op(ctx, g, tiny, O.H1_DIFFUSION, blob, assemble)
            recs.append(_probe(ctx, lambda: op.apply_add_ex(1.0, x, y)))
        prob = _h1_problem(_box(recs), p, q1d)
        x = _vector(prob.h1.ndofs, "x")
        xm = x.copy()
        xm[prob.h1.ess_dofs] = 0.0
        _H1[(p, q1d)] = (prob, common.oracle_apply(prob, O.H1_DIFFUSION, blob, x), common.oracle_apply(prob, O.H1_DIFFUSION, blob, xm))
    return (blob,) + _H1[(p, q1d)]


@pytest.mark.parametrize("assemble", [False, True], ids=["stored", "assembled"])
@pytest.mark.parametrize("p,q1d", H1_PAIRS)
def test_h1_diffusion(b2p_ctx, p, q1d, assemble):
    blob, prob, y_ref, ym = _h1_case(b2p_ctx, p, q1d)
    h1, ne = prob.h1, prob.mesh.ne
    n = h1.ndofs
    op = common.gpu_op(b2p_ctx, common.gpu_geom(b2p_ctx, prob), prob, O.H1_DIFFUSION, blob, assemble)
    x, y0 = _vector(n, "x"), _vector(n, "y0")
    xd = _dev(x)
    y = _nan(n)
    op.apply(xd, y)
    assert _rel(y.cpu().numpy(), y_ref) < RTOL
    r = _ran(b2p_ctx, H1V3, ne)
    ess = h1.ess_dofs
    op.set_essential(ess)
    ym = ym.copy()
    ym[ess] = 0.0
    yd = _dev(y0)
    op.apply_add_ex(-0.75, xd, yd, masked=True)
    assert _rel(yd.cpu().numpy(), y0 - 0.75 * ym) < RTOL
    _ran(b2p_ctx, H1V3, ne)
    if (p, q1d) == (2, 3):  # the owned | ghost split variant
        n_owned, epb = n // 2, r["elems_per_batch"]
        e1 = ne // 8 if epb == 1 else epb * (ne // (8 * epb)) + 1
        yo = torch.zeros(n_owned, dtype=torch.float64, device="cuda")
        yg = torch.zeros(n - n_owned, dtype=torch.float64, device="cuda")
        for e0, ec in ((0, e1), (e1, ne - e1)):
            op.apply_add_split(1.0, xd[:n_owned].contiguous(), xd[n_owned:].contiguous(), yo, yg, n_owned, e0, ec)
        _ran(b2p_ctx, H1V3)
        assert _rel(np.concatenate([yo.cpu().numpy(), yg.cpu().numpy()]), y_ref) < RTOL


# ------------------------------------------------------------------------------------------------------------ 3. block operators
@pytest.mark.parametrize("which", ["W", "X", "S"], ids=["weakcurl", "mixedcurl", "curlcurl_mass_weakcurl"])
@pytest.mark.parametrize("p", [2, 3, 4, 5, 6])
def test_block_operators(b2p_ctx, p, which):
    """Forward apply against the oracle; transposed apply against the cross-check kernel (B2P_APPLY_SIMPLE_KERNEL, one CTA per
    batch) at 1e-14 and by the adjoint identity <x, A^T u> = <A x, u> with the oracle's forward apply."""
    key, prob = _steady_problem(b2p_ctx, p)
    n, ne = prob.nd.ndofs, prob.mesh.ne
    op = _block_ops(b2p_ctx, prob)[which]
    if which == "S":
        y_ref = sum(c * _oracle(key, {O.CURLCURL: "K", O.ND_MASS: "M", O.ND_WEAKCURL: "W"}[k], "x") for k, c in BLOCK_SUM)
    else:
        y_ref = _oracle(key, which, "x")
    x, u = _vector(n, "x"), _vector(n, "u")
    y = _nan(n)
    op.apply(_dev(x), y)
    assert _rel(y.cpu().numpy(), y_ref) < RTOL
    _ran(b2p_ctx, _block_kernel(p), ne)
    yt = torch.zeros(n, dtype=torch.float64, device="cuda")
    op.apply_add_ex(1.0, _dev(u), yt, transpose=True)
    _ran(b2p_ctx, _block_kernel(p), ne)
    ys = torch.zeros(n, dtype=torch.float64, device="cuda")
    op.apply_add_ex(1.0, _dev(u), ys, transpose=True, simple_kernel=True)
    yt, ys = yt.cpu().numpy(), ys.cpu().numpy()
    assert np.abs(yt - ys).max() <= 1e-14 * np.abs(ys).max()
    assert abs(x @ yt - y_ref @ u) <= RTOL * np.linalg.norm(y_ref) * np.linalg.norm(u)


# ------------------------------------------------------------------------------------------------------------ 4. complex one-pass routes
def _cvec(n, re, im):
    return _vector(n, re) + 1j * _vector(n, im)


def _cmult(A, x, herm=False):
    n = x.size
    yr, yi = _nan(n), _nan(n)
    (A.mult_hermitian_transpose if herm else A.mult)(_dev(x.real), _dev(x.imag), yr, yi)
    return yr.cpu().numpy() + 1j * yi.cpu().numpy()


@pytest.mark.parametrize("p", [1, 2, 3, 4, 5, 6])
def test_complex_symmetric_sum(b2p_ctx, p):
    """K - w^2 (1 - i tan d) M + i w C with essential dofs (DIAG_ONE): one pass over the geometry for every term and both parts."""
    key, prob = _steady_problem(b2p_ctx, p)
    nd = prob.nd
    n, ne, ess = nd.ndofs, prob.mesh.ne, nd.ess_dofs
    A = _complex_sum(b2p_ctx, prob)
    assert A.fused_path() == (2 if p <= 3 else 3)
    x = _cvec(n, "x", "xi")
    Ax = {name: _oracle(key, name, "x", True) + 1j * _oracle(key, name, "xi", True) for name, _ in CPLX_SUM}
    for herm in (False, True):
        y_ref = sum((np.conj(c) if herm else c) * Ax[name] for name, c in CPLX_SUM)
        y_ref[ess] = x[ess]
        assert _rel(_cmult(A, x, herm), y_ref) < RTOL, herm
        _ran(b2p_ctx, _complex_kernel(p), ne)


_FLOQUET_BOXES = {}


@pytest.mark.parametrize("p", [2, 3, 4, 5, 6])
def test_floquet_block_sum(b2p_ctx, p):
    """The Floquet system on a z-periodic box through nd_hex_apply7_kernel<B2P_ND_BLOCK, CPLX>: mult against the per-term oracle
    applies, the Hermitian transpose by the adjoint identity <A^H u, x> = <u, A x>."""
    from palace_b200 import capi

    terms, coefs = _floquet_terms()

    def build(prob):
        g = common.gpu_geom(b2p_ctx, prob)
        ops = [common.gpu_op(b2p_ctx, g, prob, k, b) for k, b in terms]
        return capi.ComplexOperator.par(b2p_ctx, prob.nd.ndofs, prob.nd.ndofs, ops, coefs, prob.nd.ess_dofs, 1)

    if p not in _FLOQUET_BOXES:
        tiny = _tiny(p, periodic=True)
        A = build(tiny)
        xt = _cvec(tiny.nd.ndofs, "x", "xi")
        _FLOQUET_BOXES[p] = _box([_probe(b2p_ctx, lambda: _cmult(A, xt))], min_nz=3)
    prob = _problem(("floquet", p), _FLOQUET_BOXES[p], p, periodic=True)
    nd = prob.nd
    n, ne, ess = nd.ndofs, prob.mesh.ne, nd.ess_dofs
    A = build(prob)
    assert A.fused_path() == 3
    x, u = _cvec(n, "x", "xi"), _cvec(n, "u", "y0")
    xm = x.copy()
    xm[ess] = 0.0
    # reference: the real coefficients' terms as one curl-curl + mass pair (k-mass + 1.5 I), the two mixed kinds times i
    kx = cross_matrix((0.0, 0.0, 0.4))
    pair = cf.coeff_ctx_pair(cf.coeff_ctx(np.array([0]), (kx.T @ kx + 1.5 * np.eye(3))[None]), cf.coeff_ctx(a=1.0))
    ref = [(O.CURLCURL_MASS, pair, 1.0), (terms[2][0], terms[2][1], 1j), (terms[3][0], terms[3][1], 1j)]
    y_ref = sum(c * (common.oracle_apply(prob, k, b, xm.real) + 1j * common.oracle_apply(prob, k, b, xm.imag)) for k, b, c in ref)
    y_ref[ess] = x[ess]
    assert _rel(_cmult(A, x), y_ref) < RTOL
    _ran(b2p_ctx, ND7 + ":block:cplx", ne)
    h = _cmult(A, u, herm=True)
    _ran(b2p_ctx, ND7 + ":block:cplx", ne)
    assert abs(np.vdot(h, x) - np.vdot(u, y_ref)) <= RTOL * np.linalg.norm(y_ref) * np.linalg.norm(u)


# ------------------------------------------------------------------------------------------------------------ 5. PDL zero-fill
@pytest.mark.parametrize("p", PDL_ORDERS)
def test_par_operator_zero_fill_overlaps_the_element_kernel(b2p_ctx, p):
    """ParOperator::Mult with essential dofs zero-fills y by a kernel that releases its dependent at once and launches the element
    kernel with programmatic stream serialisation: y full of NaN, twice in a row into the same y."""
    key, prob = _steady_problem(b2p_ctx, p)
    nd = prob.nd
    n, ne, ess = nd.ndofs, prob.mesh.ne, nd.ess_dofs
    A = _par(b2p_ctx, prob, "KM")
    x = _vector(n, "x")
    y_ref = _oracle(key, "KM", "x", masked=True).copy()
    y_ref[ess] = x[ess]
    y = _nan(n)
    for _ in range(2):
        A.mult(_dev(x), y)
        assert _rel(y.cpu().numpy(), y_ref) < RTOL
        _ran(b2p_ctx, ND6 if p == 3 else ND7, ne)

"""The hexahedral unit cell of a z-periodic structure (hexmesh.box_mesh(..., periodic_z=True)) and the Floquet pencil on it.

1. The ND space of the periodic box is conforming across the identified z faces: the tangential trace of any field at a point
   of z = 0 equals its trace at the matching point of z = d; the essential (PEC) dofs lie on the x / y walls only.
2. The oracle's Floquet pencil on that space -- curl-curl + mass([k x]^T [k x]) + i (weak curl + mixed curl), the four terms
   and contexts of floquet_matrices in test_cylinder_floquet_golden.py -- reproduces the closed-form spectrum of a PEC
   rectangular waveguide cell with Bloch wave number kz:  (m pi / a)^2 + (n pi / b)^2 + (kz + 2 pi l / d)^2, TE and TM.
"""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import pyoracle as O
from palace_b200.host import coeff as cf
from palace_b200.host import hexmesh as hm
from palace_b200.host import hexspace as hs
from tests import common
from tests.test_cylinder_floquet_golden import cross_matrix

SIZE = (1.0, 0.8, 0.9)


def _corner_frame(mesh, e):
    """Origin and columns of the (affine part of the) map of element e: x = X0 + F xi."""
    c = mesh.corners[e] if mesh.corners is not None else mesh.verts[mesh.elems[e]]
    return c[0], np.stack([c[1] - c[0], c[2] - c[0], c[4] - c[0]], axis=1)


def _reference_field(sp_, e, xe_dofs, xi):
    """Reference-space value of the ND field with lexicographic element dofs xe_dofs at the reference point xi."""
    p = sp_.p
    op, _ = hs.gauss_legendre(p)
    cp = hs.gauss_lobatto(p + 1)
    bo = [np.asarray(hs.lagrange_table(op, [t])[0][0], dtype=float) for t in xi]
    bc = [np.asarray(hs.lagrange_table(cp, [t])[0][0], dtype=float) for t in xi]
    u = np.zeros(3)
    for l, (c, i, j, k) in enumerate(hs._nd_lex_layout(p)):
        f = [bc[0][i], bc[1][j], bc[2][k]]
        f[c] = bo[c][(i, j, k)[c]]
        u[c] += xe_dofs[l] * f[0] * f[1] * f[2]
    return u


def _tangential_trace(mesh, sp_, x, e, point):
    """(u_x, u_y) of the field x of space sp_ at a physical point on a z face of element e. On such a face the warp vanishes with
    its tangential derivatives, so the face map, and with it the tangential trace, follows from the corners alone."""
    x0, F = _corner_frame(mesh, e)
    xi = np.linalg.solve(F, point - x0)
    assert np.all(xi > -1e-12) and np.all(xi < 1 + 1e-12)
    xe_dofs = sp_.lex_sign[e] * x[sp_.lex_gid[e]]
    u = np.linalg.solve(F.T, _reference_field(sp_, e, xe_dofs, np.clip(xi, 0.0, 1.0)))  # J^-T u_ref (tangential part exact)
    return u[:2]


def _element_at(mesh, point):
    """The one element whose closure holds the point (points of a z face away from element edges)."""
    hits = []
    for e in range(mesh.ne):
        x0, F = _corner_frame(mesh, e)
        xi = np.linalg.solve(F, point - x0)
        if np.all(xi > -1e-9) and np.all(xi < 1 + 1e-9):
            hits.append(e)
    assert len(hits) == 1, (point, hits)
    return hits[0]


def _wall_faces(mesh, topo):
    """Boundary faces of the mesh; asserts that each lies on a wall x = 0, a or y = 0, b."""
    corner = lambda c: c[0] + 2 * c[1] + 4 * c[2]
    wall = np.zeros(topo.nface, bool)
    for e in range(mesh.ne):
        for nax in range(3):
            t1, t2 = [d for d in range(3) if d != nax]
            for side in range(2):
                f = topo.face_id[e, nax, side]
                if topo.face_nelem[f] != 1:
                    continue
                cs = []
                for a in range(2):
                    for b in range(2):
                        c = [0, 0, 0]
                        c[nax], c[t1], c[t2] = side, a, b
                        cs.append(mesh.corners[e, corner(c)])
                cs = np.array(cs)
                at = [np.ptp(cs[:, d]) < 1e-12 and min(abs(cs[0, d]), abs(cs[0, d] - SIZE[d])) < 1e-12 for d in range(2)]
                assert at[0] or at[1], cs
                wall[f] = True
    return wall


@pytest.mark.parametrize("p", [1, 2, 3])
def test_periodic_box_nd_space_is_conforming_across_the_z_faces(p):
    n = (3, 2, 3)
    mesh = hm.box_mesh(n, SIZE, warp_amp=0.05, scramble_seed=7, periodic_z=True)
    topo = hs.build_topology(mesh)
    nd = hs.build_nd_space(mesh, topo, p)
    rng = np.random.default_rng(1)
    x = rng.standard_normal(nd.ndofs)
    # points of the z = 0 face away from element edges, and their partners on z = d
    pts = [np.array([SIZE[0] * (i + f) / n[0], SIZE[1] * (j + g) / n[1], 0.0])
           for i in range(n[0]) for j in range(n[1]) for f, g in ((0.3, 0.6), (0.71, 0.22))]
    shift = np.array([0.0, 0.0, SIZE[2]])
    worst, scale = 0.0, 0.0
    for pt in pts:
        t0 = _tangential_trace(mesh, nd, x, _element_at(mesh, pt), pt)
        t1 = _tangential_trace(mesh, nd, x, _element_at(mesh, pt + shift), pt + shift)
        worst = max(worst, np.abs(t0 - t1).max())
        scale = max(scale, np.abs(t0).max())
    assert scale > 0.1
    assert worst < 1e-12 * scale
    # without the identification the same check fails: the two faces carry independent dofs
    plain = hm.box_mesh(n, SIZE, warp_amp=0.05, scramble_seed=7)
    nd_plain = hs.build_nd_space(plain, hs.build_topology(plain), p)
    xp = rng.standard_normal(nd_plain.ndofs)
    d = (_tangential_trace(plain, nd_plain, xp, _element_at(plain, pts[0]), pts[0])
         - _tangential_trace(plain, nd_plain, xp, _element_at(plain, pts[0] + shift), pts[0] + shift))
    assert np.abs(d).max() > 1e-3
    # the z faces are interior: the boundary faces are the 2 (ny nz + nx nz) wall faces, and the essential dofs are exactly
    # the dofs on them
    assert (topo.face_nelem == 1).sum() == 2 * (n[1] * n[2] + n[0] * n[2])
    wall = _wall_faces(mesh, topo)
    on_wall = np.zeros(nd.ndofs, bool)
    for e in range(mesh.ne):
        for l, (c, i, j, k) in enumerate(hs._nd_lex_layout(p)):
            ix = [i, j, k]
            for nax in [a for a in range(3) if a != c]:
                if ix[nax] in (0, p) and wall[topo.face_id[e, nax, ix[nax] // p]]:
                    on_wall[nd.lex_gid[e, l]] = True
    ess = np.zeros(nd.ndofs, bool)
    ess[nd.ess_dofs] = True
    assert ess.any() and (~ess).any() and np.array_equal(ess, on_wall)


def test_periodic_box_rejects_two_layers():
    with pytest.raises(ValueError):
        hm.box_mesh((2, 2, 2), periodic_z=True)


def floquet_pencil(prob, k):
    """(K_r, K_i, M) with the essential dofs removed, as floquet_matrices builds them, on the hex space of prob."""
    kx = cross_matrix(k)
    am = np.array([0])
    one = cf.coeff_ctx(a=1.0)
    A = lambda kind, blob: common.oracle_matrix(prob, kind, blob, eliminate=False)
    Kr = A(O.CURLCURL, one) + A(O.ND_MASS, cf.coeff_ctx(am, (kx.T @ kx)[None]))
    Ki = A(O.ND_WEAKCURL, cf.coeff_ctx(am, kx[None], a=-1.0)) + A(O.ND_MIXEDCURL, cf.coeff_ctx(am, kx[None], transpose=True))
    M = A(O.ND_MASS, one)
    free = np.setdiff1d(np.arange(prob.nd.ndofs), prob.nd.ess_dofs)
    sub = lambda X: X.tocsr()[free][:, free]
    return sub(Kr), sub(Ki), sub(M)


def waveguide_spectrum(kz, n_modes):
    """Lowest eigenvalues omega^2 of the PEC rectangular waveguide cell a x b x d with Bloch wave number kz, with multiplicity:
    one TE mode for each (m, n) != (0, 0) and one TM mode for m, n >= 1, at every axial harmonic l."""
    a, b, d = SIZE
    lam = []
    for m in range(6):
        for n in range(6):
            for l in range(-4, 5):
                v = (m * np.pi / a) ** 2 + (n * np.pi / b) ** 2 + (kz + 2 * np.pi * l / d) ** 2
                lam += [v] * ((m > 0 or n > 0) + (m > 0 and n > 0))
    return np.sort(lam)[:n_modes]


def pencil_eigenvalues(prob, kz, n_modes):
    Kr, Ki, M = floquet_pencil(prob, (0.0, 0.0, kz))
    assert abs(Ki + Ki.T).max() <= 1e-12 * abs(Ki).max()  # the mixed pair is skew-symmetric: K_r + i K_i is Hermitian
    # the Hermitian pencil as the real symmetric one of twice the size (every eigenvalue twice), as in the tet Floquet test
    A2 = sp.bmat([[Kr, -Ki], [Ki, Kr]], format="csc")
    M2 = sp.block_diag([M, M], format="csc")
    lam2 = common.eigsh_above(A2, M2, 2 * n_modes, 1.0, extra=8)
    assert np.abs(lam2[0::2] - lam2[1::2]).max() < 1e-8 * lam2.max()
    return 0.5 * (lam2[0::2] + lam2[1::2])


def test_floquet_pencil_on_the_periodic_hex_box_matches_the_waveguide_spectrum():
    kz, n_modes = 0.4, 11
    exact = waveguide_spectrum(kz, n_modes + 1)
    assert exact[n_modes] - exact[n_modes - 1] > 1e-2 * exact[n_modes]  # the 11 modes end at a gap of the spectrum
    exact = exact[:n_modes]
    # what the Floquet terms move: distance of every mode to the k = 0 spectrum
    at_zero = waveguide_spectrum(0.0, 60)
    dist = min(np.abs(at_zero - v).min() / v for v in exact)
    errs = {}
    for p in (2, 3, 4):
        mesh = hm.box_mesh((3, 3, 3), SIZE, scramble_seed=11, periodic_z=True)
        prob = common.problem_on_mesh(mesh, p=p, mesh_order=1)
        lam = pencil_eigenvalues(prob, kz, n_modes)
        errs[p] = np.abs(lam - exact).max() / exact.max()
    print("relative eigenvalue error by order:", errs, "distance to the kz = 0 spectrum:", dist)
    # p-convergence: each order gains at least a factor of 10, and the finest is 100x below what the Floquet terms move.
    # (Orders above 4 gain nothing more on boxes this coarse: the modes with a full half wave across one element level off near
    # 1e-5 in the plain PEC cavity of the same box too, without periodicity and without the Floquet terms.)
    assert errs[3] < 0.1 * errs[2] and errs[4] < 0.1 * errs[3]
    assert errs[4] < 1e-2 * dist

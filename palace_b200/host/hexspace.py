"""Caller-side finite element spaces on conforming hex meshes: what MFEM/Palace supply at the
drop-in boundary (SURVEY §8b "inputs available at the boundary"):

* 1-D tables (``fe.GetDofToQuad(ir, TENSOR)``-equivalent for the open/closed bases),
  /root/reference/palace/fem/libceed/basis.cpp:15-38,40-85
* the tensor-element ``GetDofMap()`` (lexicographic -> native, signed),
  /root/reference/palace/fem/libceed/restriction.cpp:134-136
* element restriction in NATIVE order with orientation signs
  (``GetElementDofs`` -> ``idx``/``orients``, restriction.cpp:281-297)
* essential (PEC) dof lists, dof multiplicities, element-local interpolation matrices for the
  p-prolongation and the discrete gradient (``GetTransferMatrix``/``ProjectGrad``,
  /root/reference/palace/fem/libceed/basis.cpp:116-165).

The global numbering is built here from a canonical per-entity orientation (edge: low -> high
global vertex; face: frame anchored at the smallest global vertex), so any conforming hex mesh,
including ones whose elements have arbitrarily rotated local frames, gets consistent signs.
"""
from __future__ import annotations

import dataclasses

import numpy as np
from numpy.polynomial import legendre as _leg

from .hexmesh import HexMesh

# --------------------------------------------------------------------------------------------
# 1-D point sets / Lagrange tables (float64; the oracle has an independent long-double version)
# --------------------------------------------------------------------------------------------


def gauss_legendre(n):
    x, w = _leg.leggauss(n)
    return 0.5 * (x + 1.0), 0.5 * w


def gauss_lobatto(n):
    if n == 2:
        return np.array([0.0, 1.0])
    c = np.zeros(n)
    c[-1] = 1.0  # P_{n-1}
    r = _leg.legroots(_leg.legder(c))
    x = np.concatenate([[-1.0], np.sort(r), [1.0]])
    # Newton polish on P'_{n-1}
    d1 = _leg.legder(c)
    d2 = _leg.legder(d1)
    for _ in range(3):
        x[1:-1] -= _leg.legval(x[1:-1], d1) / _leg.legval(x[1:-1], d2)
    x = 0.5 * (x - x[::-1])  # symmetrise
    return 0.5 * (x + 1.0)


def lagrange_table(nodes, pts):
    """B[q, j] = l_j(pts[q]), G[q, j] = l_j'(pts[q]) for the Lagrange basis through ``nodes``."""
    nodes = np.asarray(nodes, dtype=np.longdouble)
    pts = np.asarray(pts, dtype=np.longdouble)
    n = len(nodes)
    B = np.zeros((len(pts), n), dtype=np.longdouble)
    G = np.zeros((len(pts), n), dtype=np.longdouble)
    for j in range(n):
        others = [m for m in range(n) if m != j]
        den = np.prod(nodes[j] - nodes[others]) if others else np.longdouble(1)
        val = np.ones_like(pts)
        for m in others:
            val = val * (pts - nodes[m])
        der = np.zeros_like(pts)
        for k in others:
            pr = np.ones_like(pts)
            for m in others:
                if m != k:
                    pr = pr * (pts - nodes[m])
            der = der + pr
        B[:, j] = val / den
        G[:, j] = der / den
    return B.astype(np.float64), G.astype(np.float64)


@dataclasses.dataclass
class Tables1D:
    """1-D tables at the q1d Gauss-Legendre points (quadrature order 2p -> q1d = p+1 by default,
    /root/reference/palace/fem/integrator.cpp:14-22)."""

    p: int
    q1d: int
    Bo: np.ndarray  # [q1d, p]    open (Gauss-Legendre) Lagrange basis
    Bc: np.ndarray  # [q1d, p+1]  closed (Gauss-Lobatto) Lagrange basis
    Gc: np.ndarray  # [q1d, p+1]  d/dx of closed basis
    qw: np.ndarray  # [q1d]
    qx: np.ndarray  # [q1d]


def tables_1d(p, q1d=None) -> Tables1D:
    q1d = p + 1 if q1d is None else q1d
    qx, qw = gauss_legendre(q1d)
    op, _ = gauss_legendre(p)
    cp = gauss_lobatto(p + 1)
    Bo, _ = lagrange_table(op, qx)
    Bc, Gc = lagrange_table(cp, qx)
    return Tables1D(p, q1d, Bo, Bc, Gc, qw, qx)


# --------------------------------------------------------------------------------------------
# MFEM native ordering of ND_HexahedronElement (independent transcription; the oracle has its own)
# --------------------------------------------------------------------------------------------


def nd_hex_dofmap(p):
    """dof_map[lex] = native, or -1-native for a sign flip (TensorBasisElement::GetDofMap())."""
    d3 = p * (p + 1) * (p + 1)
    m = np.full(3 * d3, 10 ** 9, dtype=np.int64)
    o = 0
    X = lambda i, j, k: 0 * d3 + i + (j + k * (p + 1)) * p
    Y = lambda i, j, k: 1 * d3 + i + (j + k * p) * (p + 1)
    Z = lambda i, j, k: 2 * d3 + i + (j + k * (p + 1)) * (p + 1)
    edges = [
        lambda i: X(i, 0, 0), lambda i: Y(p, i, 0), lambda i: X(i, p, 0), lambda i: Y(0, i, 0),
        lambda i: X(i, 0, p), lambda i: Y(p, i, p), lambda i: X(i, p, p), lambda i: Y(0, i, p),
        lambda i: Z(0, 0, i), lambda i: Z(p, 0, i), lambda i: Z(p, p, i), lambda i: Z(0, p, i),
    ]
    for f in edges:
        for i in range(p):
            m[f(i)] = o
            o += 1
    # bottom (3,2,1,0)
    for j in range(1, p):
        for i in range(p):
            m[X(i, p - j, 0)] = o; o += 1
    for j in range(p):
        for i in range(1, p):
            m[Y(i, p - 1 - j, 0)] = -1 - o; o += 1
    # front (0,1,5,4)
    for k in range(1, p):
        for i in range(p):
            m[X(i, 0, k)] = o; o += 1
    for k in range(p):
        for i in range(1, p):
            m[Z(i, 0, k)] = o; o += 1
    # right (1,2,6,5)
    for k in range(1, p):
        for j in range(p):
            m[Y(p, j, k)] = o; o += 1
    for k in range(p):
        for j in range(1, p):
            m[Z(p, j, k)] = o; o += 1
    # back (2,3,7,6)
    for k in range(1, p):
        for i in range(p):
            m[X(p - 1 - i, p, k)] = -1 - o; o += 1
    for k in range(p):
        for i in range(1, p):
            m[Z(p - i, p, k)] = o; o += 1
    # left (3,0,4,7)
    for k in range(1, p):
        for j in range(p):
            m[Y(0, p - 1 - j, k)] = -1 - o; o += 1
    for k in range(p):
        for j in range(1, p):
            m[Z(0, p - j, k)] = o; o += 1
    # top (4,5,6,7)
    for j in range(1, p):
        for i in range(p):
            m[X(i, j, p)] = o; o += 1
    for j in range(p):
        for i in range(1, p):
            m[Y(i, j, p)] = o; o += 1
    # interior
    for k in range(1, p):
        for j in range(1, p):
            for i in range(p):
                m[X(i, j, k)] = o; o += 1
    for k in range(1, p):
        for j in range(p):
            for i in range(1, p):
                m[Y(i, j, k)] = o; o += 1
    for k in range(p):
        for j in range(1, p):
            for i in range(1, p):
                m[Z(i, j, k)] = o; o += 1
    assert o == 3 * d3 and (m != 10 ** 9).all()
    return m


# --------------------------------------------------------------------------------------------
# Mesh topology with canonical entity frames
# --------------------------------------------------------------------------------------------


@dataclasses.dataclass
class HexTopology:
    nv: int
    nedge: int
    nface: int
    edge_id: np.ndarray    # [NE, 3, 2, 2]  axis d, corner (u,v) of the other two axes (increasing axis order)
    edge_flip: np.ndarray  # same shape, bool: local +d direction runs high -> low global vertex
    face_id: np.ndarray    # [NE, 3, 2]     normal axis, side
    face_a0: np.ndarray    # [NE, 3, 2]     origin corner along in-face axis t1 (t1 < t2)
    face_b0: np.ndarray    # [NE, 3, 2]     origin corner along in-face axis t2
    face_swap: np.ndarray  # [NE, 3, 2]     canonical first axis is t2
    face_nelem: np.ndarray  # [nface] number of adjacent elements (1 = boundary)
    edge_verts: np.ndarray  # [nedge, 2]
    face_verts: np.ndarray  # [nface, 4] sorted


def _others(d):
    return [a for a in range(3) if a != d]


def build_topology(mesh: HexMesh) -> HexTopology:
    el = mesh.elems
    ne = el.shape[0]
    nv = int(el.max()) + 1
    corner = lambda a: a[0] + 2 * a[1] + 4 * a[2]
    # edges
    ekeys = np.empty((ne, 3, 2, 2, 2), dtype=np.int64)
    for d in range(3):
        o1, o2 = _others(d)
        for u in range(2):
            for v in range(2):
                a = [0, 0, 0]
                a[o1], a[o2] = u, v
                a[d] = 0
                ga = el[:, corner(a)]
                a[d] = 1
                gb = el[:, corner(a)]
                ekeys[:, d, u, v, 0] = ga
                ekeys[:, d, u, v, 1] = gb
    lo = ekeys.min(axis=-1)
    hi = ekeys.max(axis=-1)
    flip = ekeys[..., 0] > ekeys[..., 1]
    uniq, inv = np.unique((lo * nv + hi).ravel(), return_inverse=True)
    edge_id = inv.reshape(ne, 3, 2, 2)
    edge_verts = np.stack([uniq // nv, uniq % nv], axis=1)
    # faces
    fg = np.empty((ne, 3, 2, 2, 2), dtype=np.int64)  # [e, normal axis, side, a(t1), b(t2)]
    for n in range(3):
        t1, t2 = _others(n)
        for s in range(2):
            for a_ in range(2):
                for b_ in range(2):
                    c = [0, 0, 0]
                    c[n], c[t1], c[t2] = s, a_, b_
                    fg[:, n, s, a_, b_] = el[:, corner(c)]
    flat = fg.reshape(ne, 3, 2, 4)
    amin = flat.argmin(axis=-1)
    a0 = amin // 2
    b0 = amin % 2
    ee, nn, ss = np.meshgrid(np.arange(ne), np.arange(3), np.arange(2), indexing="ij")
    nb1 = fg[ee, nn, ss, 1 - a0, b0]
    nb2 = fg[ee, nn, ss, a0, 1 - b0]
    swap = nb2 < nb1
    srt = np.sort(flat, axis=-1).reshape(-1, 4)
    uniqf, invf, cnt = np.unique(srt, axis=0, return_inverse=True, return_counts=True)
    face_id = invf.reshape(ne, 3, 2)
    return HexTopology(
        nv=nv, nedge=len(uniq), nface=len(uniqf), edge_id=edge_id, edge_flip=flip, face_id=face_id,
        face_a0=a0, face_b0=b0, face_swap=swap, face_nelem=cnt, edge_verts=edge_verts, face_verts=uniqf,
    )


# --------------------------------------------------------------------------------------------
# Spaces
# --------------------------------------------------------------------------------------------


@dataclasses.dataclass
class HexSpace:
    kind: str               # "nd" | "h1"
    p: int
    ndofs: int              # local (L-vector) size
    P: int                  # dofs per element
    lex_gid: np.ndarray     # [NE, P] int64 global dof of each LEXICOGRAPHIC element dof
    lex_sign: np.ndarray    # [NE, P] int8 (+1/-1); all +1 for H1
    dof_map: np.ndarray     # [P] lexicographic -> native (signed); identity for H1 (Palace uses lexico there)
    ess_dofs: np.ndarray    # sorted int64 list of dofs on the boundary (PEC / Dirichlet)
    mult: np.ndarray        # [ndofs] number of elements touching each dof

    def native_restriction(self):
        """(idx[NE,P] int32, orient[NE,P] int8) in NATIVE element order, as
        InitNativeRestr builds them (restriction.cpp:281-297): u_nat[n] = orient * x[idx]."""
        ne = self.lex_gid.shape[0]
        idx = np.empty((ne, self.P), dtype=np.int32)
        ori = np.empty((ne, self.P), dtype=np.int8)
        nat = np.where(self.dof_map < 0, -1 - self.dof_map, self.dof_map)
        sgn = np.where(self.dof_map < 0, -1, 1).astype(np.int8)
        idx[:, nat] = self.lex_gid
        ori[:, nat] = self.lex_sign * sgn[None, :]
        return idx, ori


def _nd_lex_layout(p):
    """Lexicographic element dofs: list of (comp, i, j, k) in storage order."""
    out = []
    n = p + 1
    for k in range(n):
        for j in range(n):
            for i in range(p):
                out.append((0, i, j, k))
    for k in range(n):
        for j in range(p):
            for i in range(n):
                out.append((1, i, j, k))
    for k in range(p):
        for j in range(n):
            for i in range(n):
                out.append((2, i, j, k))
    return out


def build_nd_space(mesh: HexMesh, topo: HexTopology, p: int) -> HexSpace:
    ne = mesh.ne
    P = 3 * p * (p + 1) ** 2
    n_e, n_f, n_i = p, 2 * p * (p - 1), 3 * p * (p - 1) ** 2
    off_f = topo.nedge * n_e
    off_i = off_f + topo.nface * n_f
    ndofs = off_i + ne * n_i
    gid = np.empty((ne, P), dtype=np.int64)
    sgn = np.ones((ne, P), dtype=np.int8)
    earange = np.arange(ne)
    int_count = 0
    for l, (c, i, j, k) in enumerate(_nd_lex_layout(p)):
        ix = [i, j, k]
        o1, o2 = _others(c)
        b1 = ix[o1] in (0, p)
        b2 = ix[o2] in (0, p)
        io = ix[c]
        if b1 and b2:
            u, v = ix[o1] // p, ix[o2] // p
            fl = topo.edge_flip[:, c, u, v]
            gid[:, l] = topo.edge_id[:, c, u, v] * n_e + np.where(fl, p - 1 - io, io)
            sgn[:, l] = np.where(fl, -1, 1)
        elif b1 or b2:
            nax = o1 if b1 else o2          # face normal axis
            oc = o2 if b1 else o1           # the closed in-face axis
            side = ix[nax] // p
            kc = ix[oc]
            t1, t2 = _others(nax)
            a0 = topo.face_a0[:, nax, side]
            b0 = topo.face_b0[:, nax, side]
            sw = topo.face_swap[:, nax, side]
            org_c = a0 if c == t1 else b0   # origin side along the tangent axis
            org_o = a0 if oc == t1 else b0
            io_c = np.where(org_c == 1, p - 1 - io, io)
            kc_c = np.where(org_o == 1, p - kc, kc)
            first = np.where(sw, t2, t1)
            fam = np.where(first == c, 0, 1)
            loc = fam * p * (p - 1) + io_c + p * (kc_c - 1)
            gid[:, l] = off_f + topo.face_id[:, nax, side] * n_f + loc
            sgn[:, l] = np.where(org_c == 1, -1, 1)
        else:
            gid[:, l] = off_i + earange * n_i + int_count
            int_count += 1
    assert int_count == n_i
    mult = np.bincount(gid.ravel(), minlength=ndofs)
    # essential dofs: everything on boundary faces (their edges included)
    ess = np.zeros(ndofs, dtype=bool)
    bfaces = topo.face_nelem == 1
    for l, (c, i, j, k) in enumerate(_nd_lex_layout(p)):
        ix = [i, j, k]
        for nax in _others(c):
            if ix[nax] in (0, p):
                side = ix[nax] // p
                onb = bfaces[topo.face_id[:, nax, side]]
                ess[gid[onb, l]] = True
    return HexSpace("nd", p, ndofs, P, gid, sgn, nd_hex_dofmap(p), np.nonzero(ess)[0], mult)


def build_h1_space(mesh: HexMesh, topo: HexTopology, p: int) -> HexSpace:
    ne = mesh.ne
    n = p + 1
    P = n ** 3
    n_e, n_f, n_i = p - 1, (p - 1) ** 2, (p - 1) ** 3
    off_e = topo.nv
    off_f = off_e + topo.nedge * n_e
    off_i = off_f + topo.nface * n_f
    ndofs = off_i + ne * n_i
    gid = np.empty((ne, P), dtype=np.int64)
    earange = np.arange(ne)
    int_count = 0
    ess = np.zeros(ndofs, dtype=bool)
    bfaces = topo.face_nelem == 1
    for k in range(n):
        for j in range(n):
            for i in range(n):
                l = i + n * (j + n * k)
                ix = [i, j, k]
                bnd = [a for a in range(3) if ix[a] in (0, p)]
                if len(bnd) == 3:
                    gid[:, l] = mesh.elems[:, (i // p) + 2 * (j // p) + 4 * (k // p)]
                elif len(bnd) == 2:
                    d = [a for a in range(3) if a not in bnd][0]
                    o1, o2 = _others(d)
                    u, v = ix[o1] // p, ix[o2] // p
                    fl = topo.edge_flip[:, d, u, v]
                    t = ix[d]
                    gid[:, l] = off_e + topo.edge_id[:, d, u, v] * n_e + np.where(fl, p - t, t) - 1
                elif len(bnd) == 1:
                    nax = bnd[0]
                    side = ix[nax] // p
                    t1, t2 = _others(nax)
                    a0 = topo.face_a0[:, nax, side]
                    b0 = topo.face_b0[:, nax, side]
                    sw = topo.face_swap[:, nax, side]
                    u = np.where(a0 == 1, p - ix[t1], ix[t1])
                    v = np.where(b0 == 1, p - ix[t2], ix[t2])
                    s = np.where(sw, v, u)
                    t = np.where(sw, u, v)
                    gid[:, l] = off_f + topo.face_id[:, nax, side] * n_f + (s - 1) + (p - 1) * (t - 1)
                else:
                    gid[:, l] = off_i + earange * n_i + int_count
                    int_count += 1
                for nax in bnd:
                    side = ix[nax] // p
                    onb = bfaces[topo.face_id[:, nax, side]]
                    ess[gid[onb, l]] = True
    mult = np.bincount(gid.ravel(), minlength=ndofs)
    return HexSpace("h1", p, ndofs, P, gid, np.ones((ne, P), dtype=np.int8), np.arange(P, dtype=np.int64),
                    np.nonzero(ess)[0], mult)


# --------------------------------------------------------------------------------------------
# Element-local interpolation matrices (lexicographic bases), geometry independent
# --------------------------------------------------------------------------------------------


def nd_prolongation_matrix(pc: int, pf: int) -> np.ndarray:
    """I[l_f, m_c] = fine dof functional l_f applied to coarse ND shape function m_c
    (mfem GetTransferMatrix semantics used by basis.cpp:132-150), lexicographic on both sides."""
    opc, _ = gauss_legendre(pc)
    cpc = gauss_lobatto(pc + 1)
    opf, _ = gauss_legendre(pf)
    cpf = gauss_lobatto(pf + 1)
    Oo, _ = lagrange_table(opc, opf)  # [pf, pc]   coarse open basis at fine open points
    Cc, _ = lagrange_table(cpc, cpf)  # [pf+1, pc+1]
    lay_f = _nd_lex_layout(pf)
    lay_c = _nd_lex_layout(pc)
    I = np.zeros((len(lay_f), len(lay_c)))
    for lf, (c, i, j, k) in enumerate(lay_f):
        for mc, (c2, i2, j2, k2) in enumerate(lay_c):
            if c != c2:
                continue
            tx = Oo[i, i2] if c == 0 else Cc[i, i2]
            ty = Oo[j, j2] if c == 1 else Cc[j, j2]
            tz = Oo[k, k2] if c == 2 else Cc[k, k2]
            I[lf, mc] = tx * ty * tz
    return I


def h1_prolongation_matrix(pc: int, pf: int) -> np.ndarray:
    cpc = gauss_lobatto(pc + 1)
    cpf = gauss_lobatto(pf + 1)
    C, _ = lagrange_table(cpc, cpf)
    return np.einsum("kc,jb,ia->kjicba", C, C, C).reshape((pf + 1) ** 3, (pc + 1) ** 3)


def discrete_gradient_matrix(p: int) -> np.ndarray:
    """G[l_nd, m_h1] = tangential derivative of H1 shape m at ND node l (mfem ProjectGrad)."""
    op, _ = gauss_legendre(p)
    cp = gauss_lobatto(p + 1)
    _, dC = lagrange_table(cp, op)  # [p, p+1] closed-basis derivative at open points
    n = p + 1
    lay = _nd_lex_layout(p)
    G = np.zeros((len(lay), n ** 3))
    for l, (c, i, j, k) in enumerate(lay):
        ix = [i, j, k]
        for t in range(n):
            m = list(ix)
            m[c] = t
            G[l, m[0] + n * (m[1] + n * m[2])] = dC[ix[c], t]
    return G


# --------------------------------------------------------------------------------------------
# Raviart-Thomas space RT_{p-1} on hexahedra (the H(div) partner of ND_p: curl ND_p is contained in RT_{p-1}); used by the
# flux error estimator (/root/reference/palace/linalg/errorestimator.cpp: B = curl E lives in the RT space of
# RT_FECollection(p - 1)). Component c is CLOSED (p + 1 Gauss-Lobatto nodes) along axis c and OPEN (p Gauss-Legendre nodes) along
# the other two; reference-to-physical map u = J u^ / det J.
# --------------------------------------------------------------------------------------------


def _rt_lex_layout(p):
    """Lexicographic element dofs: list of (comp, i, j, k) in storage order (i fastest)."""
    out = []
    for c in range(3):
        n = [p, p, p]
        n[c] = p + 1
        for k in range(n[2]):
            for j in range(n[1]):
                for i in range(n[0]):
                    out.append((c, i, j, k))
    return out


def _perm_sign(t1, t2, n):
    """+1 if (t1, t2, n) is an even permutation of (0, 1, 2)."""
    return 1 if (t1, t2, n) in ((0, 1, 2), (1, 2, 0), (2, 0, 1)) else -1


def build_rt_space(mesh: HexMesh, topo: HexTopology, p: int) -> HexSpace:
    """Face dofs: p^2 normal-flux dofs per face in the face's canonical frame (origin = smallest vertex id, first axis towards
    its smaller neighbour), positive along first x second; an element sees them with the sign of its local +n axis against
    that normal (elements are positively oriented). Interior dofs: 3 p^2 (p - 1) per element."""
    ne = mesh.ne
    lay = _rt_lex_layout(p)
    P = len(lay)
    n_f, n_i = p * p, 3 * p * p * (p - 1)
    off_i = topo.nface * n_f
    ndofs = off_i + ne * n_i
    gid = np.empty((ne, P), dtype=np.int64)
    sgn = np.ones((ne, P), dtype=np.int8)
    earange = np.arange(ne)
    int_count = 0
    ess = np.zeros(ndofs, dtype=bool)
    bfaces = topo.face_nelem == 1
    for l, (c, i, j, k) in enumerate(lay):
        ix = [i, j, k]
        if ix[c] in (0, p):
            side = ix[c] // p
            t1, t2 = _others(c)
            a0 = topo.face_a0[:, c, side]
            b0 = topo.face_b0[:, c, side]
            sw = topo.face_swap[:, c, side]
            u = np.where(a0 == 1, p - 1 - ix[t1], ix[t1])
            v = np.where(b0 == 1, p - 1 - ix[t2], ix[t2])
            s = np.where(sw, v, u)
            t = np.where(sw, u, v)
            gid[:, l] = topo.face_id[:, c, side] * n_f + s + p * t
            # canonical normal = (+-e_t1) x (+-e_t2), exchanged under swap; e_t1 x e_t2 = perm(t1, t2, c) e_c
            sg = _perm_sign(t1, t2, c) * np.where(a0 == 1, -1, 1) * np.where(b0 == 1, -1, 1) * np.where(sw, -1, 1)
            sgn[:, l] = sg
            onb = bfaces[topo.face_id[:, c, side]]
            ess[gid[onb, l]] = True
        else:
            gid[:, l] = off_i + earange * n_i + int_count
            int_count += 1
    assert int_count == n_i
    mult = np.bincount(gid.ravel(), minlength=ndofs)
    return HexSpace("rt", p, ndofs, P, gid, sgn, np.arange(P, dtype=np.int64), np.nonzero(ess)[0], mult)


def rt_prolongation_matrix(pc: int, pf: int) -> np.ndarray:
    """I[l_f, m_c] = fine RT dof functional l_f applied to coarse RT shape function m_c (GetTransferMatrix semantics), lexicographic on
    both sides: per component, closed (Gauss-Lobatto) interpolation along its own axis and open (Gauss-Legendre) along the other two
    -- ND's assignment (nd_prolongation_matrix) with the roles exchanged."""
    opc, _ = gauss_legendre(pc)
    cpc = gauss_lobatto(pc + 1)
    opf, _ = gauss_legendre(pf)
    cpf = gauss_lobatto(pf + 1)
    Oo, _ = lagrange_table(opc, opf)  # [pf, pc]
    Cc, _ = lagrange_table(cpc, cpf)  # [pf+1, pc+1]
    lay_f = _rt_lex_layout(pf)
    lay_c = _rt_lex_layout(pc)
    I = np.zeros((len(lay_f), len(lay_c)))
    for lf, (c, i, j, k) in enumerate(lay_f):
        for mc, (c2, i2, j2, k2) in enumerate(lay_c):
            if c != c2:
                continue
            tx = Cc[i, i2] if c == 0 else Oo[i, i2]
            ty = Cc[j, j2] if c == 1 else Oo[j, j2]
            tz = Cc[k, k2] if c == 2 else Oo[k, k2]
            I[lf, mc] = tx * ty * tz
    return I


def rt_hex_dense_interp(p: int, q1d: int) -> np.ndarray:
    """interp[3][Q][P]: reference-space values of the lexicographic RT basis at the tensor Gauss-Legendre points (x fastest),
    the layout of libCEED non-tensor bases (fem/libceed/basis.cpp:40-85)."""
    t = tables_1d(p, q1d)
    lay = _rt_lex_layout(p)
    Q = q1d ** 3
    out = np.zeros((3, Q, len(lay)))
    for l, (c, i, j, k) in enumerate(lay):
        tx = t.Bc[:, i] if c == 0 else t.Bo[:, i]
        ty = t.Bc[:, j] if c == 1 else t.Bo[:, j]
        tz = t.Bc[:, k] if c == 2 else t.Bo[:, k]
        out[c, :, l] = np.einsum("c,b,a->cba", tz, ty, tx).ravel()
    return out


def nd_hex_dense_interp(p: int, q1d: int) -> np.ndarray:
    """interp[3][Q][P] of the LEXICOGRAPHIC ND basis (open along the component's axis, closed along the others)."""
    t = tables_1d(p, q1d)
    lay = _nd_lex_layout(p)
    Q = q1d ** 3
    out = np.zeros((3, Q, len(lay)))
    for l, (c, i, j, k) in enumerate(lay):
        tx = t.Bo[:, i] if c == 0 else t.Bc[:, i]
        ty = t.Bo[:, j] if c == 1 else t.Bc[:, j]
        tz = t.Bo[:, k] if c == 2 else t.Bc[:, k]
        out[c, :, l] = np.einsum("c,b,a->cba", tz, ty, tx).ravel()
    return out


def discrete_curl_matrix(p: int) -> np.ndarray:
    """C[l_rt, m_nd]: the curl of ND shape function m expanded in the RT basis (both lexicographic), mfem ProjectCurl
    semantics: (curl u)_c = d_a u_b - d_b u_a for (c, a, b) cyclic; the derivative of the closed basis along an axis is exactly
    representable in the open basis of that axis (values at the Gauss-Legendre nodes)."""
    op, _ = gauss_legendre(p)
    cp = gauss_lobatto(p + 1)
    _, dC = lagrange_table(cp, op)  # [p, p+1] closed-basis derivative at the open points
    lay_nd = _nd_lex_layout(p)
    rt_index = {key: l for l, key in enumerate(_rt_lex_layout(p))}
    C = np.zeros((len(rt_index), len(lay_nd)))
    for m, (b, i, j, k) in enumerate(lay_nd):          # ND function with component b
        ix = [i, j, k]
        for a in range(3):                             # derivative direction a != b
            if a == b:
                continue
            c = 3 - a - b                              # the curl component that receives d_a u_b
            sign = 1.0 if (c, a, b) in ((0, 1, 2), (1, 2, 0), (2, 0, 1)) else -1.0
            # u_b is closed along a (a != b): d_a maps the closed index ix[a] onto the open indices along a; it stays open
            # along b and closed along c -- exactly the RT component c layout
            for t in range(p):
                tgt = list(ix)
                tgt[a] = t
                C[rt_index[(c, tgt[0], tgt[1], tgt[2])], m] += sign * dC[t, ix[a]]
    return C

"""Conforming hexahedral meshes for the synthetic configurations (caller-side stand-in for the
mfem::ParMesh Palace hands to ``BilinearForm::PartialAssemble``,
/root/reference/palace/fem/bilinearform.cpp:27-107 and /root/reference/palace/fem/mesh.cpp:146-209).

Local vertex numbering follows MFEM's hexahedron: vertex ``v`` at reference corner
``((1,0,0),(1,1,0),(0,1,0) ...)``; ``LEX2MFEM[a + 2 b + 4 c]`` gives the MFEM local vertex at
lattice corner ``(a, b, c)``.
"""
from __future__ import annotations

import dataclasses

import numpy as np

LEX2MFEM = np.array([0, 1, 3, 2, 4, 5, 7, 6], dtype=np.int64)
MFEM2LEX = np.argsort(LEX2MFEM)

# 12 edges as pairs of lattice corners (lexicographic corner id a+2b+4c), grouped by direction.
# faces as (axis, side).


def _rotations():
    """The 24 orientation-preserving symmetries of the cube as permutations of lattice corners."""
    import itertools

    rots = []
    for perm in itertools.permutations(range(3)):
        for flips in itertools.product([0, 1], repeat=3):
            # map new reference coords xi' -> old reference coords: old[perm[d]] = flip? 1-xi'[d] : xi'[d]
            M = np.zeros((3, 3))
            for d in range(3):
                M[perm[d], d] = -1.0 if flips[d] else 1.0
            if np.linalg.det(M) < 0:
                continue
            rots.append((perm, flips))
    return rots


_ROTS = _rotations()


@dataclasses.dataclass
class HexMesh:
    """``elems[e, a+2b+4c]`` = global vertex at lattice corner (a,b,c) of element e (LEXICOGRAPHIC
    corner order; convert with LEX2MFEM for MFEM's local numbering)."""

    verts: np.ndarray  # [NV, 3] straight-sided vertex coordinates (before warp)
    elems: np.ndarray  # [NE, 8] int64
    attr: np.ndarray  # [NE] int32, 1-based, contiguous (mesh.cpp:46-83)
    warp: object = None  # optional smooth map R^3 -> R^3 applied to all node coordinates
    # [NE, 8, 3] physical corner coordinates when they are not verts[elems]: a periodic mesh identifies the vertices of
    # opposite faces in `elems` (the connectivity the spaces are numbered from), while each element keeps its own corners.
    # Code that takes element positions from verts[elems] (element centroids for partitioning, for instance) sees the top
    # layer of a periodic mesh folded onto the bottom face: read the corners through node_coords / `corners` instead.
    corners: np.ndarray = None

    @property
    def ne(self):
        return self.elems.shape[0]

    def node_coords(self, order: int, nodes1d: np.ndarray) -> np.ndarray:
        """Element node coordinates xe[NE, 3, (order+1)^3] at the tensor lattice ``nodes1d`` (x
        fastest), component-major like mfem::Ordering::byNODES (/root/reference/palace/fem/mesh.hpp:31-33)."""
        n = order + 1
        assert len(nodes1d) == n
        t = np.asarray(nodes1d, dtype=np.float64)
        X, Y, Z = np.meshgrid(t, t, t, indexing="ij")  # [i,j,k]
        # flatten x fastest
        xi = np.stack([X.transpose(2, 1, 0).ravel(), Y.transpose(2, 1, 0).ravel(), Z.transpose(2, 1, 0).ravel()])
        w = np.empty((8, n ** 3))
        for c in range(2):
            for b in range(2):
                for a in range(2):
                    w[a + 2 * b + 4 * c] = (
                        (xi[0] if a else 1 - xi[0]) * (xi[1] if b else 1 - xi[1]) * (xi[2] if c else 1 - xi[2])
                    )
        vc = self.verts[self.elems] if self.corners is None else self.corners  # [NE, 8, 3]
        xe = np.einsum("evc,vn->ecn", vc, w)
        if self.warp is not None:
            xe = self.warp(xe)
        return np.ascontiguousarray(xe)


def box_mesh(n, size=(1.0, 1.0, 1.0), *, warp_amp=0.0, scramble_seed=None, n_attr=1, origin=(0.0, 0.0, 0.0),
             periodic_z=False) -> HexMesh:
    """Uniform nx*ny*nz box. ``warp_amp`` > 0 applies a smooth non-affine warp to every node
    (SURVEY §8d.2 'smoothly warped variant'); ``scramble_seed`` rotates each element's local frame
    by a random cube symmetry so that edge/face orientation handling is exercised; attributes are
    striped ``1 + e % n_attr`` (test/unit/test-libceed.cpp:54-64).

    ``periodic_z``: the unit cell of a structure periodic along z (Floquet-periodic models). The vertices of the top face are
    the bottom face's in the connectivity, so the two z faces are interior and the spaces are continuous across them; the
    elements keep their physical corners (``HexMesh.corners``). The warp vanishes on both z faces, so it keeps them matching.
    Needs nz >= 3: with two layers the vertical edges of both layers would join the same two vertices."""
    if np.isscalar(n):
        n = (int(n),) * 3
    nx, ny, nz = n
    if periodic_z and nz < 3:
        raise ValueError(f"periodic_z needs at least 3 element layers along z, got nz = {nz}")
    xs = origin[0] + np.linspace(0, size[0], nx + 1)
    ys = origin[1] + np.linspace(0, size[1], ny + 1)
    zs = origin[2] + np.linspace(0, size[2], nz + 1)
    vid = lambda i, j, k: i + (nx + 1) * (j + (ny + 1) * k)
    K, J, I = np.meshgrid(np.arange(nz + 1), np.arange(ny + 1), np.arange(nx + 1), indexing="ij")
    verts = np.stack([xs[I.ravel()], ys[J.ravel()], zs[K.ravel()]], axis=1)
    ek, ej, ei = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    ei, ej, ek = ei.ravel(), ej.ravel(), ek.ravel()
    elems = np.empty((ei.size, 8), dtype=np.int64)
    for c in range(2):
        for b in range(2):
            for a in range(2):
                elems[:, a + 2 * b + 4 * c] = vid(ei + a, ej + b, ek + c)
    if scramble_seed is not None:
        rng = np.random.default_rng(scramble_seed)
        choice = rng.integers(0, len(_ROTS), size=elems.shape[0])
        new = np.empty_like(elems)
        for r, (perm, flips) in enumerate(_ROTS):
            sel = np.nonzero(choice == r)[0]
            if sel.size == 0:
                continue
            for c in range(2):
                for b in range(2):
                    for a in range(2):
                        newc = (a, b, c)
                        old = [0, 0, 0]
                        for d in range(3):
                            old[perm[d]] = 1 - newc[d] if flips[d] else newc[d]
                        new[sel, a + 2 * b + 4 * c] = elems[sel, old[0] + 2 * old[1] + 4 * old[2]]
        elems = new
    corners = None
    if periodic_z:
        corners = verts[elems]
        layer = (nx + 1) * (ny + 1)
        elems = np.where(elems >= nz * layer, elems - nz * layer, elems)  # top vertex layer -> bottom vertex layer
    attr = (1 + (np.arange(elems.shape[0]) % n_attr)).astype(np.int32)
    warp = None
    if warp_amp:
        L = np.array(size, dtype=np.float64)
        o = np.array(origin, dtype=np.float64)

        def warp(xe, amp=warp_amp, L=L, o=o):
            # xe [..., 3, n]; boundary-preserving smooth perturbation
            s = (xe - o[None, :, None]) / L[None, :, None]
            sx, sy, sz = s[:, 0], s[:, 1], s[:, 2]
            bump = np.sin(np.pi * sx) * np.sin(np.pi * sy) * np.sin(np.pi * sz)
            out = xe.copy()
            out[:, 0] += amp * L[0] * bump * np.cos(2.0 * sy + 0.3)
            out[:, 1] += amp * L[1] * bump * np.sin(1.7 * sz + 0.1)
            out[:, 2] += amp * L[2] * bump * np.cos(1.3 * sx - 0.2)
            return out

    return HexMesh(verts=verts, elems=elems, attr=attr, warp=warp, corners=corners)


def partition_box(n, parts):
    """Element -> rank map for a uniform box of ``n`` elements split into a ``parts`` = (px,py,pz)
    block grid (stand-in for mesh::Partition, /root/reference/palace/driver.cpp:66-70)."""
    if np.isscalar(n):
        n = (int(n),) * 3
    nx, ny, nz = n
    px, py, pz = parts
    ek, ej, ei = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    bi = (ei.ravel() * px) // nx
    bj = (ej.ravel() * py) // ny
    bk = (ek.ravel() * pz) // nz
    return (bi + px * (bj + py * bk)).astype(np.int32)

"""Generates tests/golden/spheres_mesh.npz from the REFERENCE's spheres example mesh (run where the reference tree is available;
pass its root as the first argument): examples/spheres/mesh/spheres.msh, 14,362 cubic tetrahedra (TET20). The file itself is
3.4 MB, so the fixture keeps what the mesh needs and nothing more:
  * the corner vertices, corner connectivity, attributes and boundary triangles, as gmsh.load_tets returns them;
  * the nodes (lattice order, gmsh.load_tets's xe) that sit off the affine image of their element's corners, as one table of
    unique positions and an index per CURVED element (-1 for its affine nodes) -- 12,698 of the 14,362 elements are affine
    (every node within 1e-15 of the element size of its affine image), and tests/test_spheres_golden.py rebuilds every
    affine node from the corners.
The mesh rebuilt from the fixture is checked against gmsh.load_tets of the original file before it is written."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from palace_b200.host import gmsh  # noqa: E402
from tests.test_spheres_golden import affine_nodes, load_fixture  # noqa: E402


def main(ref):
    m = gmsh.load_tets(os.path.join(ref, "examples/spheres/mesh/spheres.msh"))
    X = np.transpose(m.xe, (0, 2, 1))                                     # [ne][Nn][3]
    h = np.linalg.norm(m.verts[m.elems[:, 1:]] - m.verts[m.elems[:, :1]], axis=2).max(axis=1)
    off = np.abs(X - affine_nodes(m.verts, m.elems, m.order)).max(axis=2) > 1e-13 * h[:, None]   # [ne][Nn]
    curved = np.flatnonzero(off.any(axis=1))
    nodes, inv = np.unique(X[off], axis=0, return_inverse=True)
    idx = np.full(off.shape, -1, dtype=np.int64)
    idx[off] = inv.ravel()
    idx = idx[curved]
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "spheres_mesh.npz")
    np.savez_compressed(path, order=m.order, verts=m.verts, elems=m.elems.astype(np.int32), attr=m.attr,
                        bdr_verts=m.bdr_verts.astype(np.int32), bdr_attr=m.bdr_attr, curved=curved.astype(np.int32),
                        curved_nodes=nodes, curved_idx=idx.astype(np.int32))
    r = load_fixture(path)
    assert np.abs(r.xe - m.xe).max() < 1e-14 * np.abs(m.xe).max()
    assert all((getattr(r, k) == getattr(m, k)).all() for k in ("verts", "elems", "attr", "bdr_verts", "bdr_attr"))
    print("wrote", path, os.path.getsize(path), "bytes;", m.ne, "tets,", curved.size, "curved,", nodes.shape[0], "nodes off their affine positions")


if __name__ == "__main__":
    main(sys.argv[1])

"""CPU: the Raviart-Thomas p-prolongation on hexahedra (hexspace.rt_prolongation_matrix and its Kronecker factors
assemble.rt_prolongation_comps, the tables b2p_interp_create takes): exact on every coarse field, conforming across shared faces of
scrambled, warped meshes, and a Galerkin hierarchy for the RT mass (P^T M_f P = M_c with the oracle's H(div) mass matrices)."""
import numpy as np
import pytest

from oracle import estimator as E
from oracle import solvers as S
from palace_b200.host import assemble as asm
from palace_b200.host import hexmesh as hm
from palace_b200.host import hexspace as hs
from tests.common import problem_on_mesh

PAIRS = [(1, 2), (2, 4), (1, 4), (2, 3), (3, 6)]


def _kron_from_comps(comps, P_out, P_in):
    I = np.zeros((P_out, P_in))
    for cc in comps:
        Ax, Ay, Az = cc["A"]
        blk = np.kron(Az, np.kron(Ay, Ax))  # x fastest on both sides
        no, ni = int(np.prod(cc["out_n"])), int(np.prod(cc["in_n"]))
        I[cc["out_off"]:cc["out_off"] + no, cc["in_off"]:cc["in_off"] + ni] = blk
    return I


@pytest.mark.parametrize("pc,pf", PAIRS)
def test_prolongation_comps_reproduce_the_matrix(pc, pf):
    I = hs.rt_prolongation_matrix(pc, pf)
    assert I.shape == (3 * pf * pf * (pf + 1), 3 * pc * pc * (pc + 1))
    assert np.abs(_kron_from_comps(asm.rt_prolongation_comps(pc, pf), *I.shape) - I).max() < 1e-14


@pytest.mark.parametrize("pc,pf", PAIRS)
def test_prolongated_field_equals_the_coarse_field_at_the_points(pc, pf):
    q1d = pf + 1
    I = hs.rt_prolongation_matrix(pc, pf)
    Bf, Bc = hs.rt_hex_dense_interp(pf, q1d), hs.rt_hex_dense_interp(pc, q1d)
    assert np.abs(np.einsum("cqf,fm->cqm", Bf, I) - Bc).max() < 1e-13


def _mesh():
    return hm.box_mesh((3, 2, 2), (1.0, 0.7, 0.9), warp_amp=0.04, scramble_seed=5, n_attr=3)


@pytest.mark.parametrize("pc,pf", [(1, 2), (2, 4), (1, 3)])
def test_shared_face_dofs_agree(pc, pf):
    mesh = _mesh()
    topo = hs.build_topology(mesh)
    sc, sf = hs.build_rt_space(mesh, topo, pc), hs.build_rt_space(mesh, topo, pf)
    I = hs.rt_prolongation_matrix(pc, pf)
    x = np.random.default_rng(3).standard_normal(sc.ndofs)
    val = np.full(sf.ndofs, np.nan)
    for e in range(mesh.ne):
        yf = sf.lex_sign[e] * (I @ (sc.lex_sign[e] * x[sc.lex_gid[e]]))  # global-orientation values of the fine dofs
        seen = ~np.isnan(val[sf.lex_gid[e]])
        assert np.abs(val[sf.lex_gid[e]][seen] - yf[seen]).max(initial=0.0) < 1e-12 * max(1.0, np.abs(yf).max())
        val[sf.lex_gid[e]] = yf
    assert not np.isnan(val).any()


def _rt_mass(prob, sp, coef_elem):
    B = E.rt_hex_tables(sp.p, prob.q1d)
    return E.mixed_mass_matrix(prob.qdata_ref, B, E.HDIV, sp.lex_gid, sp.lex_sign.astype(float), sp.ndofs, B, E.HDIV, sp.lex_gid,
                               sp.lex_sign.astype(float), sp.ndofs, coef_elem)


@pytest.mark.parametrize("pc,pf", [(1, 2), (2, 4)])
def test_galerkin_identity_of_the_rt_mass(pc, pf):
    mesh = _mesh()
    prob = problem_on_mesh(mesh, p=pf)
    sc, sf = hs.build_rt_space(mesh, prob.topo, pc), hs.build_rt_space(mesh, prob.topo, pf)
    rng = np.random.default_rng(11)
    G = rng.standard_normal((3, 3, 3))
    mats = np.einsum("kij,klj->kil", G, G) + 2.0 * np.eye(3)[None]  # anisotropic SPD per attribute
    coef_elem = mats[mesh.attr - 1]
    Mf, Mc = _rt_mass(prob, sf, coef_elem), _rt_mass(prob, sc, coef_elem)
    P = S.interp_matrix(hs.rt_prolongation_matrix(pc, pf), sc.lex_gid, sc.lex_sign.astype(float), sf.lex_gid, sf.lex_sign.astype(float),
                        sc.ndofs, sf.ndofs)
    R = (P.T @ Mf @ P - Mc).toarray()
    assert np.abs(R).max() < 1e-13 * abs(Mc).max()

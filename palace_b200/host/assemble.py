"""Caller-side glue that turns host spaces (hexspace.HexSpace) into C-ABI descriptors: the stand-in
for BilinearForm::PartialAssemble / Assemble(hierarchy) and the DiscreteLinearOperator assembly
(/root/reference/palace/fem/bilinearform.cpp:27-107,155-200,203-282) and for
fem::ConstructFECollections' p-sequence (/root/reference/palace/fem/multigrid.hpp:23-73)."""
from __future__ import annotations

import numpy as np

from . import hexspace as hs


def p_sequence(p, coarsen="logarithmic", pmin=1):
    """Orders of the p-multigrid hierarchy, coarse -> fine (multigrid.hpp:44-70)."""
    seq = [p]
    while seq[-1] > pmin:
        q = seq[-1]
        seq.append((q + pmin) // 2 if coarsen == "logarithmic" else q - 1)
    return seq[::-1]


def space_dict(sp: hs.HexSpace):
    if sp.kind == "nd":
        idx, ori = sp.native_restriction()
        return dict(P=sp.P, lsize=sp.ndofs, idx=idx, orient=ori, dof_map=sp.dof_map)
    if sp.kind == "rt":  # lexicographic is native here; the face dofs carry their orientation sign
        return dict(P=sp.P, lsize=sp.ndofs, idx=sp.lex_gid.astype(np.int32), orient=sp.lex_sign, dof_map=None)
    return dict(P=sp.P, lsize=sp.ndofs, idx=sp.lex_gid.astype(np.int32), orient=None, dof_map=None)


def nd_prolongation_comps(pc, pf):
    """Kronecker factors of the ND hex p-prolongation (GetTransferMatrix semantics): per vector
    component, open-basis interpolation along its own axis and closed-basis along the others."""
    opc, _ = hs.gauss_legendre(pc)
    cpc = hs.gauss_lobatto(pc + 1)
    opf, _ = hs.gauss_legendre(pf)
    cpf = hs.gauss_lobatto(pf + 1)
    Oo, _ = hs.lagrange_table(opc, opf)  # [pf, pc]
    Cc, _ = hs.lagrange_table(cpc, cpf)  # [pf+1, pc+1]
    nc, nf = pc + 1, pf + 1
    d3c, d3f = pc * nc * nc, pf * nf * nf
    comps = []
    for c in range(3):
        in_n = [nc] * 3
        out_n = [nf] * 3
        in_n[c], out_n[c] = pc, pf
        A = [Cc, Cc, Cc]
        A[c] = Oo
        comps.append(dict(in_off=c * d3c, in_n=in_n, out_off=c * d3f, out_n=out_n, A=A))
    return comps


def rt_prolongation_comps(pc, pf):
    """Kronecker factors of the RT hex p-prolongation (hexspace.rt_prolongation_matrix): per vector component, closed-basis
    interpolation along its own axis and open-basis along the other two."""
    opc, _ = hs.gauss_legendre(pc)
    cpc = hs.gauss_lobatto(pc + 1)
    opf, _ = hs.gauss_legendre(pf)
    cpf = hs.gauss_lobatto(pf + 1)
    Oo, _ = hs.lagrange_table(opc, opf)  # [pf, pc]
    Cc, _ = hs.lagrange_table(cpc, cpf)  # [pf+1, pc+1]
    d3c, d3f = (pc + 1) * pc * pc, (pf + 1) * pf * pf
    comps = []
    for c in range(3):
        in_n = [pc] * 3
        out_n = [pf] * 3
        in_n[c], out_n[c] = pc + 1, pf + 1
        A = [Oo, Oo, Oo]
        A[c] = Cc
        comps.append(dict(in_off=c * d3c, in_n=in_n, out_off=c * d3f, out_n=out_n, A=A))
    return comps


def h1_prolongation_comps(pc, pf):
    cpc = hs.gauss_lobatto(pc + 1)
    cpf = hs.gauss_lobatto(pf + 1)
    Cc, _ = hs.lagrange_table(cpc, cpf)
    return [dict(in_off=0, in_n=[pc + 1] * 3, out_off=0, out_n=[pf + 1] * 3, A=[Cc, Cc, Cc])]


def curl_table(p):
    """D [p][p+1]: derivative of the closed (Gauss-Lobatto) 1-D basis at the open (Gauss-Legendre) nodes, the 1-D factor of the
    discrete gradient (ProjectGrad) and of the discrete curl (ProjectCurl) on hexahedra."""
    op, _ = hs.gauss_legendre(p)
    cp = hs.gauss_lobatto(p + 1)
    return hs.lagrange_table(cp, op)[1]


def gradient_comps(p):
    """Kronecker factors of the discrete gradient H1(p) -> ND(p) (ProjectGrad): derivative of the
    closed basis at the open points along the component's axis, identity along the others."""
    dC = curl_table(p)  # [p, p+1]
    n = p + 1
    I = np.eye(n)
    d3 = p * n * n
    comps = []
    for c in range(3):
        out_n = [n] * 3
        out_n[c] = p
        A = [I, I, I]
        A[c] = dC
        comps.append(dict(in_off=0, in_n=[n] * 3, out_off=c * d3, out_n=out_n, A=A))
    return comps


def curl_kron_terms(p):
    """The discrete curl ND(p) -> RT(p-1) as two sums of Kronecker factors, one per term of RT_c = D_a u_b - D_b u_a ((c, a, b)
    cyclic): the form two b2p_interp_create handles applied one after the other take. Interp.curl_hex applies both terms in one
    pass; this form is its cross-check."""
    D = curl_table(p)
    n = p + 1
    Ip, In = np.eye(p), np.eye(n)
    d3_nd, d3_rt = p * n * n, n * p * p
    terms = [[], []]
    for c in range(3):
        a, b = (c + 1) % 3, (c + 2) % 3
        out_n = [p] * 3
        out_n[c] = n
        for t, (src, ax, sign) in enumerate(((b, a, 1.0), (a, b, -1.0))):  # + D_a u_b, - D_b u_a
            in_n = [n] * 3
            in_n[src] = p
            A = [None] * 3
            A[ax] = sign * D
            A[src] = Ip
            A[c] = In
            terms[t].append(dict(in_off=src * d3_nd, in_n=in_n, out_off=c * d3_rt, out_n=out_n, A=A))
    return terms

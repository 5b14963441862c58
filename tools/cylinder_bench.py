#!/usr/bin/env python
"""BASELINE configs 0 / 2 on the reference's own geometry: eigenmodes of the cylinder cavity (examples/cylinder/cavity_pec.json,
HEX27 mesh from tests/golden/cylinder_cavity_pec.npz, optionally uniformly refined) through the device stack -- ARPACK
shift-invert over FGMRES + p-multigrid (LOGARITHMIC coarsening) + Chebyshev/Hiptmair. Reports sizes, setup and solve times,
operator / V-cycle timings and the eigenfrequencies next to the reference's stored values (level 0) and the closed forms.
GPU box:  python tools/cylinder_bench.py --order 4 --refine 2 --nev 4 [--coarse ams]      (refine 3 at order 4 = 7.9M dofs)"""
import argparse
import json
import os
import sys
import time

import numpy as np
import scipy.sparse.linalg as spla
from scipy.special import jn_zeros, jnp_zeros

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def analytic_ghz(count, a=2.74e-2, d=5.48e-2, eps_r=2.08):
    c = 299792458.0 / np.sqrt(eps_r)
    f = []
    for n in range(0, 6):
        for m, (pe, pm) in enumerate(zip(jnp_zeros(n, 4), jn_zeros(n, 4)), start=1):
            for l in range(0, 5):
                mult = 1 if n == 0 else 2
                if l >= 1:
                    f += [c / (2 * np.pi) * np.sqrt((pe / a) ** 2 + (l * np.pi / d) ** 2)] * mult   # TE_nml
                f += [c / (2 * np.pi) * np.sqrt((pm / a) ** 2 + (l * np.pi / d) ** 2)] * mult        # TM_nml
    return np.sort(f)[:count] / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--order", type=int, default=4)
    ap.add_argument("--refine", type=int, default=0)
    ap.add_argument("--nev", type=int, default=4)
    ap.add_argument("--tol", type=float, default=1e-10)
    ap.add_argument("--coarse-tol", type=float, default=1e-10, help="relative tolerance of the coarse-level PCG (the reference's coarse solve is one AMS V-cycle)")
    ap.add_argument("--coarse", choices=["pcg", "ams"], default="pcg",
                    help="coarse solver: Jacobi-PCG to --coarse-tol, or AMS on the assembled p=1 matrix with the reference's defaults "
                         "(cycle_it = order, mg_cycle_it = 2)")
    ap.add_argument("--cheby-order", type=int, default=0, help="Chebyshev smoother order; 0 = the reference's default max(2p, 4) (iodata.cpp:533-536)")
    args = ap.parse_args()
    import torch

    from oracle import pyoracle as O  # noqa: F401  (tests.common imports it)
    from palace_b200 import capi
    from palace_b200.host import assemble as asm
    from palace_b200.host import coeff as cf
    from palace_b200.host import gmsh
    from palace_b200.host import hexspace as hs
    from tests import common
    from tests.test_cylinder_golden import FIX, frequencies_ghz, target_lambda

    t0 = time.time()
    m = gmsh.Hex27Mesh(FIX["verts"], FIX["elems"], FIX["attr"], np.ascontiguousarray(FIX["xe2"]), FIX["bdr_attr"], FIX["bdr_verts"])
    for _ in range(args.refine):
        m = gmsh.refine_hex27(m)
    p = args.order
    topo = hs.build_topology(m)
    orders = asm.p_sequence(p)
    nd = {q: hs.build_nd_space(m, topo, q) for q in orders}
    h1 = {q: hs.build_h1_space(m, topo, q) for q in orders}
    q1d = p + 1
    nodes = hs.gauss_lobatto(3)
    qx, _ = hs.gauss_legendre(q1d)
    nB, nG = hs.lagrange_table(nodes, qx)
    m.attr = np.ones(m.ne, dtype=np.int32)
    prob = common.Problem(m, topo, p, q1d, 2, m.xe2, nd[p], h1[p], hs.tables_1d(p, q1d), (nB, nG), None)
    t_host = time.time() - t0
    ctx = capi.Ctx(0)
    capi.set_stream(ctx)
    t0 = time.time()
    geom = common.gpu_geom(ctx, prob)
    sigma = target_lambda()
    ident = cf.coeff_ctx()
    blob_A = cf.coeff_ctx_pair(cf.coeff_ctx(a=-sigma), cf.coeff_ctx(a=1.0))
    blob_P = cf.coeff_ctx_pair(cf.coeff_ctx(a=+sigma), cf.coeff_ctx(a=1.0))
    A = common.gpu_par_operator(ctx, geom, prob, O.CURLCURL_MASS, blob_A, space=nd[p])
    M = common.gpu_par_operator(ctx, geom, prob, O.ND_MASS, ident, space=nd[p])
    Pl, AG = {}, {}
    Pl[p] = common.gpu_par_operator(ctx, geom, prob, O.CURLCURL_MASS, blob_P, space=nd[p])
    AG[p] = common.gpu_par_operator(ctx, geom, prob, O.H1_DIFFUSION, cf.coeff_ctx(a=sigma), space=h1[p])
    for q in orders[:-1]:
        Pl[q] = common.gpu_par_operator(ctx, geom, prob, O.CURLCURL_MASS, blob_P, space=nd[q], fine_op=Pl[p].local_op)
        AG[q] = common.gpu_par_operator(ctx, geom, prob, O.H1_DIFFUSION, cf.coeff_ctx(a=sigma), space=h1[q], fine_op=AG[p].local_op)
    G = [common.gpu_interp(ctx, h1[q], nd[q], asm.gradient_comps(q)) for q in orders]
    P = [common.gpu_interp(ctx, nd[a], nd[b], asm.nd_prolongation_comps(a, b)) for a, b in zip(orders[:-1], orders[1:])]
    q0 = orders[0]

    def make_coarse():
        if args.coarse == "ams":
            # vertex coordinates: the corners of the second-order element nodes (lexicographic, 3 per direction)
            X = np.zeros((h1[q0].ndofs, 3))
            for c in range(8):
                X[np.asarray(m.elems)[:, c]] = np.asarray(m.xe2)[:, :, 2 * (c & 1) + 6 * ((c >> 1) & 1) + 18 * ((c >> 2) & 1)]
            Gh = common.oracle_interp(h1[q0], nd[q0], hs.discrete_gradient_matrix(1))
            return capi.Solver.assembled(ctx, capi.Solver.ams(ctx, Gh, X, cycle_it=p)), None
        c = capi.Solver.krylov(ctx, capi.CG, rel_tol=args.coarse_tol, max_it=5000)
        cj = capi.Solver.jacobi(ctx)
        c.set_check_interval(int(os.environ.get("B2P_COARSE_CG_CHECK", "8")))  # device-resident CG scalars
        if os.environ.get("B2P_COARSE_ASSEMBLED", "0") == "1":  # PCG on the device-assembled p = 1 matrix (MfemWrapperSolver flow)
            return capi.Solver.assembled(ctx, c, cj), cj
        cj.set_operator(Pl[q0])
        c.set_preconditioner(cj)
        c.set_operator(Pl[q0])
        return c, cj

    coarse, _cj = make_coarse()
    cheby_order = args.cheby_order if args.cheby_order > 0 else max(2 * p, 4)
    mg_cycle_it = 2 if args.coarse == "ams" else 1
    mg = capi.Solver.gmg(ctx, coarse, P, G, cycle_it=mg_cycle_it, smooth_it=1, cheby_order=cheby_order)
    mg.gmg_set_operators([Pl[q] for q in orders], [AG[q] for q in orders])
    ksp = capi.Solver.krylov(ctx, capi.FGMRES, rel_tol=args.tol, max_it=300, max_dim=300)
    ksp.set_operator(A)
    ksp.set_preconditioner(mg)
    torch.cuda.synchronize()
    t_setup = time.time() - t0

    n = nd[p].ndofs
    free = np.setdiff1d(np.arange(n), nd[p].ess_dofs)
    xd = torch.zeros(n, dtype=torch.float64, device="cuda")
    yd = torch.zeros(n, dtype=torch.float64, device="cuda")

    def timeit(fn, reps=20):
        fn()
        torch.cuda.synchronize()
        t = time.time()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        return (time.time() - t) / reps * 1e3

    apply_ms = timeit(lambda: A.mult(xd, yd))
    # the pieces of one V-cycle, timed alone: level operators, Hiptmair auxiliary operators, transfer operators
    level_ms = {}
    for q in orders:
        vq = torch.rand(nd[q].ndofs, dtype=torch.float64, device="cuda")
        wq = torch.empty_like(vq)
        level_ms[f"A_p{q}"] = timeit(lambda: Pl[q].mult(vq, wq))
        hq = torch.rand(h1[q].ndofs, dtype=torch.float64, device="cuda")
        gq = torch.empty_like(hq)
        level_ms[f"AG_p{q}"] = timeit(lambda: AG[q].mult(hq, gq))
        level_ms[f"G_p{q}"] = timeit(lambda: G[orders.index(q)].mult(hq, wq))
    for (a, b), Pab in zip(zip(orders[:-1], orders[1:]), P):
        va = torch.rand(nd[a].ndofs, dtype=torch.float64, device="cuda")
        vb = torch.empty(nd[b].ndofs, dtype=torch.float64, device="cuda")
        level_ms[f"P_p{a}_p{b}"] = timeit(lambda: Pab.mult(va, vb))
    xd.copy_(torch.rand(n, dtype=torch.float64))
    vcycle_ms = timeit(lambda: mg.mult(xd, yd), reps=5)
    c_in = torch.rand(nd[q0].ndofs, dtype=torch.float64, device="cuda")
    c_in[torch.from_numpy(np.asarray(nd[q0].ess_dofs, dtype=np.int64)).cuda()] = 0.0
    c_out = torch.zeros_like(c_in)
    # the multigrid owns its coarse solver: time a second one built the same way on the same level operator
    solo, _solo_cj = make_coarse()
    t = time.time()
    solo.set_operator(Pl[q0])
    torch.cuda.synchronize()
    level_ms["coarse_set_operator_ms"] = (time.time() - t) * 1e3
    level_ms["coarse_solve"] = timeit(lambda: solo.mult(c_in, c_out), reps=3)
    if args.coarse == "ams":
        level_ms["coarse_host_setup_ms"] = solo.setup_ms()
        level_ms["coarse_ams_levels"] = [solo.levels(h)[0] for h in range(4)]
    elif os.environ.get("B2P_COARSE_ASSEMBLED", "0") != "1":  # (the assembled wrapper keeps no Krylov statistics)
        level_ms["coarse_solve_its"] = solo.stats()["its"]
    its, t_solve = [], [0.0]

    def to_full(v):
        f = np.zeros(n)
        f[free] = v
        return f

    def opinv(v):
        t = time.time()
        xd.copy_(torch.from_numpy(to_full(v)))
        ksp.mult(xd, yd)
        its.append(ksp.stats()["its"])
        out = yd.cpu().numpy()[free]
        t_solve[0] += time.time() - t
        return out

    def mmul(v):
        xd.copy_(torch.from_numpy(to_full(v)))
        M.mult(xd, yd)
        return yd.cpu().numpy()[free]

    nf = free.size
    t0 = time.time()
    lam = spla.eigsh(spla.LinearOperator((nf, nf), matvec=lambda v: None, dtype=np.float64), k=args.nev,
                     M=spla.LinearOperator((nf, nf), matvec=mmul, dtype=np.float64), sigma=sigma, which="LA",
                     OPinv=spla.LinearOperator((nf, nf), matvec=opinv, dtype=np.float64), tol=max(args.tol, 1e-11),
                     v0=np.random.default_rng(0).standard_normal(nf), return_eigenvectors=False)
    t_eig = time.time() - t0
    f = frequencies_ghz(np.sort(lam)).real
    out = {"workload": f"cylinder cavity eigenmodes, ND order {p}, {m.ne} HEX27 elements (refine {args.refine})", "dofs": int(n),
           "levels": orders, "cheby_order": cheby_order, "coarse_tol": args.coarse_tol, "mg_cycle_it": mg_cycle_it,
           "coarse_level": (f"AMS (cycle_it {p}) on the device-assembled p=1 matrix" if args.coarse == "ams" else
                            "Jacobi-PCG on the device-assembled p=1 matrix" if os.environ.get("B2P_COARSE_ASSEMBLED", "0") == "1" else
                            "Jacobi-PCG, matrix-free p=1 operator"), "level_dofs": {f"nd_p{q}": int(nd[q].ndofs) for q in orders},
           "piece_ms": level_ms, "host_build_s": t_host, "device_setup_s": t_setup, "apply_ms": apply_ms, "apply_MDoF_s": n / apply_ms / 1e3,
           "vcycle_ms": vcycle_ms, "eigensolve_s": t_eig, "linear_solves": len(its), "fgmres_its_per_solve": float(np.mean(its)),
           "time_in_linear_solves_s": t_solve[0], "f_ghz": f.tolist(), "analytic_ghz": analytic_ghz(args.nev).tolist()}
    ref = FIX["ref_f_re_ghz"][: args.nev]
    if args.refine == 0 and p == int(FIX["order"]):
        out["rel_err_vs_reference_eig_csv"] = (np.abs(f - ref) / ref).tolist()
    else:
        # a finer discretisation than the one behind the stored numbers: the difference is the reference mesh's
        # discretisation error, not a parity measure
        out["rel_diff_vs_reference_eig_csv_level0"] = (np.abs(f - ref) / ref).tolist()
    out["rel_err_vs_closed_form"] = (np.abs(f - analytic_ghz(args.nev)) / analytic_ghz(args.nev)).tolist()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

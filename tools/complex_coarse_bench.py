#!/usr/bin/env python
"""Coarse level of the complex p-multigrid, three ways, on two problems:

  floquet  the z-periodic hex box with the Floquet terms, K_r + i K_i - sigma M (unit materials, k = (0, 0, kz))
  lossy    a hex cavity K - w2 (1 - i tan d) M (PEC walls)

each preconditioned by the complex p-multigrid over orders {1, 2, 3} (4th-kind Chebyshev smoothing) inside FGMRES, with the
coarsest level (p = 1) solved by
  mf     GMRES on the matrix-free complex operator with complex Jacobi (what b2p_csolver_gmg did before)
  sum    b2p_csolver_assembled, Ar + Ai: real GMRES + Jacobi on the device-assembled matrix, once per part
  block  b2p_csolver_assembled, the real 2n block [[Ar, Ai], [Ai, -Ar]]: real GMRES + Jacobi, one solve
all to the same relative tolerance (--coarse-tol).

Prints one JSON line per (problem, arm): FGMRES iterations, ms per FGMRES solve and per V-cycle (CUDA events, median of
--rounds alternated rounds after a warm-up solve), the assembly time of the coarse matrix (first set_operator: symbolic and
numeric phase; second: numeric only), the coarse matrix's size and entries, the relative difference of the solution to the mf
arm's, and the card name and power limit read in the same run.

  python tools/complex_coarse_bench.py [--n 6] [--rounds 2] [--coarse-tol 1e-6] [--coarse-restart 50]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

from oracle import pyoracle as O  # noqa: E402
from palace_b200 import capi  # noqa: E402
from palace_b200.host import assemble as asm  # noqa: E402
from palace_b200.host import coeff as cf  # noqa: E402
from palace_b200.host import hexmesh as hm  # noqa: E402
from palace_b200.host import hexspace as hs  # noqa: E402
from tests import common  # noqa: E402

ORDERS = [1, 2, 3]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def problem(name, n, kz, sigma, w2, tand):
    if name == "floquet":
        mesh = hm.box_mesh((n, n, n), (1.0, 1.0, 1.0), periodic_z=True)
        kx = np.array([[0.0, -kz, 0.0], [kz, 0.0, 0.0], [0.0, 0.0, 0.0]])
        am = np.array([0])
        one = cf.coeff_ctx(a=1.0)
        terms = [(O.CURLCURL, one), (O.ND_MASS, cf.coeff_ctx(am, (kx.T @ kx)[None])), (O.ND_WEAKCURL, cf.coeff_ctx(am, kx[None], a=-1.0)),
                 (O.ND_MIXEDCURL, cf.coeff_ctx(am, kx[None], transpose=True)), (O.ND_MASS, one)]
        coefs = [1.0, 1.0, 1j, 1j, -sigma]
    else:
        mesh = hm.box_mesh((n, n, n), (1.0, 1.0, 1.0))
        one = cf.coeff_ctx(a=1.0)
        terms = [(O.CURLCURL, one), (O.ND_MASS, one)]
        coefs = [1.0, -w2 * (1.0 - 1j * tand)]
    prob = common.problem_on_mesh(mesh, p=ORDERS[-1], mesh_order=1)
    return prob, terms, coefs


def levels(ctx, prob, terms, coefs):
    nd = {p: hs.build_nd_space(prob.mesh, prob.topo, p) for p in ORDERS}
    geom = common.gpu_geom(ctx, prob)
    fine = [common.gpu_op(ctx, geom, prob, k, b) for k, b in terms]
    A, keep = {}, [geom, fine]
    for p in ORDERS:
        sp_ = nd[p]
        if p == ORDERS[-1]:
            ops = fine
        else:
            t = hs.tables_1d(p, prob.q1d)
            idx, ori = sp_.native_restriction()
            ops = [o.coarsen(p, sp_.ndofs, idx, ori, sp_.dof_map, t.Bo, t.Bc, t.Gc) for o in fine]
            keep.append(ops)
        A[p] = capi.ComplexOperator.par(ctx, sp_.ndofs, sp_.ndofs, ops, coefs, sp_.ess_dofs, diag_policy=1)
    P = [common.gpu_interp(ctx, nd[a], nd[b], asm.nd_prolongation_comps(a, b)) for a, b in zip(ORDERS[:-1], ORDERS[1:])]
    return nd, A, P, keep


def coarse_solver(ctx, arm, tol, max_it, restart):
    """GMRES(restart) with classical Gram-Schmidt twice (one host synchronisation per orthogonalisation) in every arm."""
    if arm == "mf":
        s = capi.ComplexSolver.krylov(ctx, capi.GMRES, rel_tol=tol, max_it=max_it, max_dim=restart, orthog=capi.CGS2)
        pc = capi.ComplexSolver.jacobi(ctx, omega=1.0)
        s.set_preconditioner(pc)
        return s
    inner = capi.Solver.krylov(ctx, capi.GMRES, rel_tol=tol, max_it=max_it, max_dim=restart, orthog=capi.CGS2)
    return capi.ComplexSolver.assembled(ctx, inner, capi.Solver.jacobi(ctx), complex_matrix=(arm == "block"))


def events(torch, fn, reps=1, warm=True):
    if warm:
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--problems", nargs="+", default=["floquet", "lossy"])
    ap.add_argument("--n", type=int, default=6, help="elements per side of the box")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--vcycles", type=int, default=10, help="V-cycles per timed window")
    ap.add_argument("--coarse-tol", type=float, default=1e-6)
    ap.add_argument("--coarse-max-it", type=int, default=500)
    ap.add_argument("--coarse-restart", type=int, default=50)
    ap.add_argument("--kz", type=float, default=0.4)
    ap.add_argument("--sigma", type=float, default=-1.0)
    ap.add_argument("--w2", type=float, default=-2.0, help="w2 < 0: positive definite real part (Chebyshev smoothing)")
    ap.add_argument("--tand", type=float, default=0.1)
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "complex_coarse_bench.py measures on the GPU; there is no CPU path"
    ctx = capi.Ctx(0)
    capi.set_stream(ctx)
    name = card()
    arms = ["mf", "sum", "block"]
    for pname in args.problems:
        prob, terms, coefs = problem(pname, args.n, args.kz, args.sigma, args.w2, args.tand)
        nd, A, P, keep = levels(ctx, prob, terms, coefs)
        top = ORDERS[-1]
        n = nd[top].ndofs
        rng = np.random.default_rng(2024)
        b = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        b[nd[top].ess_dofs] = 0.0
        br, bi = torch.from_numpy(b.real.copy()).cuda(), torch.from_numpy(b.imag.copy()).cuda()
        setup = {}
        for arm in arms:
            assembly = [None, None]
            if arm != "mf":  # the coarse matrix alone: first set_operator (symbolic + numeric), then numeric only
                coarse_solver(ctx, arm, args.coarse_tol, args.coarse_max_it, args.coarse_restart).set_operator(A[ORDERS[0]])  # loads the kernels
                s = coarse_solver(ctx, arm, args.coarse_tol, args.coarse_max_it, args.coarse_restart)
                assembly = [events(torch, lambda: s.set_operator(A[ORDERS[0]]), warm=False),
                            events(torch, lambda: s.set_operator(A[ORDERS[0]]), 3)]
            coarse = coarse_solver(ctx, arm, args.coarse_tol, args.coarse_max_it, args.coarse_restart)
            mg = capi.ComplexSolver.gmg(ctx, coarse, P, None, cycle_it=1, smooth_it=1, cheby_order=4)
            mg.gmg_set_operators([A[p] for p in ORDERS])
            Ks = capi.ComplexSolver.krylov(ctx, capi.FGMRES, rel_tol=1e-8, max_it=200, max_dim=200)
            Ks.set_operator(A[top])
            Ks.set_preconditioner(mg)
            setup[arm] = dict(mg=mg, Ks=Ks, assembly=assembly, xr=torch.zeros_like(br), xi=torch.zeros_like(bi),
                              vr=torch.zeros_like(br), vi=torch.zeros_like(bi))
        ms_solve, ms_vcycle = {a: [] for a in arms}, {a: [] for a in arms}
        for _ in range(args.rounds):  # alternate the arms
            for arm in arms:
                d = setup[arm]
                ms_solve[arm].append(events(torch, lambda: d["Ks"].mult(br, bi, d["xr"], d["xi"])))
                ms_vcycle[arm].append(events(torch, lambda: d["mg"].mult(br, bi, d["vr"], d["vi"]), args.vcycles))
        ref = setup["mf"]["xr"].cpu().numpy() + 1j * setup["mf"]["xi"].cpu().numpy()
        for arm in arms:
            d = setup[arm]
            x = d["xr"].cpu().numpy() + 1j * d["xi"].cpu().numpy()
            st = d["Ks"].stats()
            print(json.dumps({"problem": pname, "arm": arm, "ndofs": int(n), "ne": int(prob.mesh.ne), "coarse_ndofs": int(nd[ORDERS[0]].ndofs),
                              "coarse_nnz": d["mg"].assembled_nnz(), "fgmres_its": st["its"], "converged": st["converged"],
                              "ms_per_solve": round(float(np.median(ms_solve[arm])), 3), "ms_solve_all": [round(v, 3) for v in ms_solve[arm]],
                              "ms_per_vcycle": round(float(np.median(ms_vcycle[arm])), 3),
                              "ms_vcycle_all": [round(v, 3) for v in ms_vcycle[arm]],
                              "assembly_ms_first": None if d["assembly"][0] is None else round(d["assembly"][0], 3),
                              "assembly_ms_again": None if d["assembly"][1] is None else round(d["assembly"][1], 3),
                              "rel_diff_vs_mf": float(np.linalg.norm(x - ref) / np.linalg.norm(ref)), "gpu": name}), flush=True)
        del setup, A, P, keep
    ctx.close()


if __name__ == "__main__":
    main()

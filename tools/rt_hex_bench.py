#!/usr/bin/env python
"""Raviart-Thomas mass on hexahedra: the dense-table operator (b2p_operator_vecfe_mass) against the sum-factorised one (B2P_RT_MASS,
flux_hex_mixed7_kernel with RT as trial and test space), alternated in one process at about 2M RT dofs, and the grad-flux projection
of one cylinder-cavity mode with Jacobi PCG against multigrid PCG.

  apply       p = 2 ... 6 at q1d = p + 1 on an n^3 box: ms per Mult (CUDA events around each Mult, L2 flushed before it, median over
              the rounds of the per-round means), algorithmic bytes per Mult (x and y per unique dof, a 4-byte index per element dof,
              80 bytes of q-data per point, a 144-byte coefficient block per element; the dense arm adds its table once) and their
              fraction of 3.35 TB/s, and the relative difference between the arms' outputs on the same seeded x
  projection  the cavity of tests/test_zzcylinder_indicator_gpu.py at order 4, first mode: FluxProjector::Mult of the grad-flux
              estimator with the sum-factorised RT mass, Jacobi PCG vs the RT p-multigrid (levels of assemble.p_sequence, coarse
              level solved on its device-assembled matrix); iterations and ms per projection (median of --reps)

Prints one JSON line per measurement with the card's name, power limit and max SM clock read in the same run.
  python tools/rt_hex_bench.py [--orders 2 3 4 5 6] [--reps 20] [--rounds 5] [--skip-projection]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

from palace_b200 import capi  # noqa: E402
from palace_b200.host import assemble as asm  # noqa: E402
from palace_b200.host import coeff as cf  # noqa: E402
from palace_b200.host import hexmesh as hm  # noqa: E402
from palace_b200.host import hexspace as hs  # noqa: E402
from tests import common  # noqa: E402

HBM = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def box_side(p, target=2.0e6):
    """elements per side for about `target` RT dofs (3 p^2 (p + 1) per element, shared faces counted once)"""
    return max(2, int(round((target / (3 * p * p * p)) ** (1.0 / 3.0))))


def time_mult(A, x, y, flush, reps, torch):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        flush.zero_()
        a.record()
        A.mult(x, y)
        b.record()
    torch.cuda.synchronize()
    return float(np.mean([a.elapsed_time(b) for a, b in ev]))


def apply_bench(ctx, p, reps, rounds, flush, name, torch):
    n1 = box_side(p)
    mesh = hm.box_mesh((n1, n1, n1), (1.0, 1.0, 1.0), n_attr=1)
    prob = common.problem_on_mesh(mesh, p=p, mesh_order=1)
    rt = hs.build_rt_space(mesh, prob.topo, p)
    geom = common.gpu_geom(ctx, prob)
    t = prob.tabs
    op = capi.Op.create(ctx, geom, capi.RT_MASS, p, rt.ndofs, rt.lex_gid, rt.lex_sign, None, t.Bo, t.Bc, None, cf.coeff_ctx(a=1.0))
    interp = hs.rt_hex_dense_interp(p, prob.q1d)
    arms = {
        "dense": capi.vecfe_mass_operator(ctx, geom, dict(P=rt.P, map_type=capi.MAP_HDIV, interp=interp, idx=rt.lex_gid, orient=rt.lex_sign,
                                                          lsize=rt.ndofs)),
        "sum_factorised": capi.Operator.par(ctx, rt.ndofs, rt.ndofs, [op]),
    }
    x = torch.from_numpy(np.random.default_rng(2024).standard_normal(rt.ndofs)).cuda()
    y = torch.empty_like(x)
    out, ms = {}, {a: [] for a in arms}
    for a, A in arms.items():
        A.mult(x, y)  # warm-up: module load, first launches
        torch.cuda.synchronize()
        out[a] = y.cpu().numpy()
    for _ in range(rounds):  # alternate the arms
        for a, A in arms.items():
            ms[a].append(time_mult(A, x, y, flush, reps, torch))
    base = op.algorithmic_bytes()
    for a in arms:
        m = float(np.median(ms[a]))
        nb = base + (8 * interp.size if a == "dense" else 0)
        print(json.dumps({"bench": "apply", "order": p, "arm": a, "ndofs": int(rt.ndofs), "ne": int(mesh.ne), "q1d": int(prob.q1d),
                          "ms_per_mult": round(m, 4), "ms_rounds": [round(v, 4) for v in ms[a]], "bytes_per_mult": int(nb),
                          "frac_of_3.35TB/s": round(nb / (m * 1e-3) / HBM, 3),
                          "rel_diff_vs_sum_factorised": float(np.linalg.norm(out[a] - out["sum_factorised"]) / np.linalg.norm(out["sum_factorised"])),
                          "speedup_of_sum_factorised": round(m / float(np.median(ms["sum_factorised"])), 3), "gpu": name}), flush=True)


def projection_bench(ctx, reps, name, torch):
    from tests.test_cylinder_indicator_golden import cavity_modes

    p = 4
    c = cavity_modes(p)
    mesh, topo, nd, rt, q1d, eps = c["mesh"], c["topo"], c["nd"], c["rt"], c["q1d"], c["eps"]
    geom = capi.Geom.from_qdata(ctx, c["qd"], q1d)
    t = hs.tables_1d(p, q1d)
    rop = capi.Op.create(ctx, geom, capi.RT_MASS, p, rt.ndofs, rt.lex_gid, rt.lex_sign, None, t.Bo, t.Bc, None, cf.coeff_ctx(a=1.0))
    Mrt = capi.Operator.par(ctx, rt.ndofs, rt.ndofs, [rop])
    sp_rt = dict(P=rt.P, map_type=capi.MAP_HDIV, interp=hs.rt_hex_dense_interp(p, q1d), idx=rt.lex_gid, orient=rt.lex_sign, lsize=rt.ndofs)
    sp_nd = dict(P=nd.P, map_type=capi.MAP_HCURL, interp=hs.nd_hex_dense_interp(p, q1d), idx=nd.lex_gid, orient=nd.lex_sign, lsize=nd.ndofs)
    I9 = np.eye(3).ravel()[None]
    orders = asm.p_sequence(p)
    spaces = [hs.build_rt_space(mesh, topo, q) for q in orders[:-1]] + [rt]
    coarse = []
    for s in spaces[:-1]:
        tt = hs.tables_1d(s.p, q1d)
        coarse.append(capi.Operator.par(ctx, s.ndofs, s.ndofs, [rop.coarsen(s.p, s.ndofs, s.lex_gid, s.lex_sign, None, tt.Bo, tt.Bc, None)]))
    P = [common.gpu_interp(ctx, a, b, asm.rt_prolongation_comps(x, y)) for a, b, x, y in zip(spaces[:-1], spaces[1:], orders[:-1], orders[1:])]
    v = torch.from_numpy(np.ascontiguousarray(c["modes"][0])).cuda()
    D = torch.zeros(rt.ndofs, dtype=torch.float64, device="cuda")
    res = {}
    for arm in ("jacobi", "multigrid"):
        est = capi.FluxEstimator(ctx, geom, sp_nd, sp_rt, eps * I9, np.sqrt(eps) * I9, I9 / np.sqrt(eps), Mrt, tol=1e-12, max_it=20000)
        if arm == "multigrid":
            est.set_multigrid(coarse + [Mrt], P, coarse_type=1, coarse_tol=1e-8, coarse_max_it=2000)
        est.project(v, D)  # warm-up
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            est.project(v, D)
            torch.cuda.synchronize()
            ts.append(1e3 * (time.perf_counter() - t0))
        st = est.stats()
        res[arm] = D.cpu().numpy()
        print(json.dumps({"bench": "projection", "order": p, "arm": arm, "levels": orders if arm == "multigrid" else [p],
                          "ndofs": int(rt.ndofs), "ne": int(mesh.ne), "iterations": st["its"], "converged": st["converged"],
                          "ms_per_projection": round(float(np.median(ts)), 3), "gpu": name}), flush=True)
    print(json.dumps({"bench": "projection", "rel_diff_multigrid_vs_jacobi":
                      float(np.linalg.norm(res["multigrid"] - res["jacobi"]) / np.linalg.norm(res["jacobi"])), "gpu": name}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--orders", type=int, nargs="+", default=[2, 3, 4, 5, 6])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-projection", action="store_true")
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "rt_hex_bench.py measures on the GPU; there is no CPU path"
    ctx = capi.Ctx(0)
    capi.set_stream(ctx)
    name = card()
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")  # larger than the 50 MB L2
    for p in args.orders:
        apply_bench(ctx, p, args.reps, args.rounds, flush, name, torch)
    if not args.skip_projection:
        projection_bench(ctx, max(3, args.reps // 4), name, torch)


if __name__ == "__main__":
    main()

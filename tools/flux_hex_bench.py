#!/usr/bin/env python
"""Flux error estimator on hexahedra: the dense-table estimator (b2p_flux_estimator_create) against the sum-factorised one
(b2p_flux_estimator_create_hex, b2p_hex_flux.cu), alternated in one process at about 2M RT dofs on an n^3 box, p = 2 ... 6 at
q1d = p + 1. Both arms share the smooth-space mass operator (sum-factorised ND or RT mass) and its p-multigrid.

  flux_mult   ms per b2p_flux_estimator_flux_mult in both directions: RT -> ND (curl-flux) and ND -> RT (grad-flux)
  integrate   ms per b2p_flux_estimator_integrate of the curl-flux (flux RT, smooth ND) and grad-flux (flux ND, smooth RT)
              configurations
  indicator   ms per b2p_flux_estimator_indicator of one real field: multigrid-preconditioned projection + integral + square root

flux_mult and integrate: CUDA events around each call, L2 flushed before it, median over the rounds of the per-round means.
indicator: wall clock of one synchronised call, L2 flushed before it, median over the rounds. Algorithmic bytes per call: x and y
once per unique dof, a 4-byte index per element dof of each space read, 80 bytes of q-data per point, the per-element coefficient
blocks of the tensor arm (80 bytes for Flux, 144 for the integral) and 16 bytes per element estimate; the dense arm adds its
[3][Q][P] tables once. The fraction is of 3.35 TB/s. rel_diff compares the two arms' outputs on the same seeded inputs.

Prints one JSON line per measurement with the card's name, power limit and max SM clock read in the same run.
  python tools/flux_hex_bench.py [--orders 2 3 4 5 6] [--reps 10] [--rounds 5] [--skip-indicator]
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


def time_calls(fn, flush, reps, torch):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        flush.zero_()
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return float(np.mean([a.elapsed_time(b) for a, b in ev]))


def levels(ctx, mesh, topo, space, fine, fine_op, M, q1d, orders):
    if space == "rt":
        spaces = [hs.build_rt_space(mesh, topo, q) for q in orders[:-1]] + [fine]
        ops = []
        for s in spaces[:-1]:
            tt = hs.tables_1d(s.p, q1d)
            ops.append(capi.Operator.par(ctx, s.ndofs, s.ndofs, [fine_op.coarsen(s.p, s.ndofs, s.lex_gid, s.lex_sign, None, tt.Bo, tt.Bc, None)]))
        comps = asm.rt_prolongation_comps
    else:
        spaces = [hs.build_nd_space(mesh, topo, q) for q in orders[:-1]] + [fine]
        ops = []
        for s in spaces[:-1]:
            idx, ori = s.native_restriction()
            tt = hs.tables_1d(s.p, q1d)
            ops.append(capi.Operator.par(ctx, s.ndofs, s.ndofs, [fine_op.coarsen(s.p, s.ndofs, idx, ori, s.dof_map, tt.Bo, tt.Bc, tt.Gc)]))
        comps = asm.nd_prolongation_comps
    P = [common.gpu_interp(ctx, a, b, comps(x, y)) for a, b, x, y in zip(spaces[:-1], spaces[1:], orders[:-1], orders[1:])]
    return ops + [M], P


def bench_order(ctx, p, reps, rounds, flush, name, torch, skip_indicator):
    n1 = box_side(p)
    mesh = hm.box_mesh((n1, n1, n1), (1.0, 1.0, 1.0), n_attr=1)
    prob = common.problem_on_mesh(mesh, p=p, mesh_order=1)
    q1d, ne, Q = prob.q1d, mesh.ne, prob.q1d ** 3
    nd, rt = prob.nd, hs.build_rt_space(mesh, prob.topo, p)
    geom = common.gpu_geom(ctx, prob)
    t = prob.tabs
    idx, ori = nd.native_restriction()
    mop = capi.Op.create(ctx, geom, capi.ND_MASS, p, nd.ndofs, idx, ori, nd.dof_map, t.Bo, t.Bc, t.Gc, cf.coeff_ctx(a=1.0))
    rop = capi.Op.create(ctx, geom, capi.RT_MASS, p, rt.ndofs, rt.lex_gid, rt.lex_sign, None, t.Bo, t.Bc, None, cf.coeff_ctx(a=1.0))
    M = {"nd": capi.Operator.par(ctx, nd.ndofs, nd.ndofs, [mop]), "rt": capi.Operator.par(ctx, rt.ndofs, rt.ndofs, [rop])}
    tens = {"nd": dict(kind=capi.ND_MASS, p=p, lsize=nd.ndofs, idx=idx, orient=ori, dof_map=nd.dof_map, Bo=t.Bo, Bc=t.Bc),
            "rt": dict(kind=capi.RT_MASS, p=p, lsize=rt.ndofs, idx=rt.lex_gid, orient=rt.lex_sign, Bo=t.Bo, Bc=t.Bc)}
    interp = {"nd": hs.nd_hex_dense_interp(p, q1d), "rt": hs.rt_hex_dense_interp(p, q1d)}
    dense = {"nd": dict(P=nd.P, map_type=capi.MAP_HCURL, interp=interp["nd"], idx=nd.lex_gid, orient=nd.lex_sign, lsize=nd.ndofs),
             "rt": dict(P=rt.P, map_type=capi.MAP_HDIV, interp=interp["rt"], idx=rt.lex_gid, orient=rt.lex_sign, lsize=rt.ndofs)}
    n = {"nd": nd.ndofs, "rt": rt.ndofs}
    Pe = {"nd": nd.P, "rt": rt.P}
    # an anisotropic, non-symmetric flux coefficient and SPD disc / smooth coefficients (one attribute)
    C = (np.eye(3) + 0.2 * np.random.default_rng(1).standard_normal((3, 3))).ravel(order="F")[None]
    S = np.diag([1.0, 2.0, 3.0])
    Cd, Cs = np.sqrt(S).ravel(order="F")[None], np.diag(1.0 / np.sqrt([1.0, 2.0, 3.0])).ravel(order="F")[None]
    rng = np.random.default_rng(2024)
    x = {s: torch.from_numpy(rng.standard_normal(n[s])).cuda() for s in ("nd", "rt")}
    orders = asm.p_sequence(p)
    common_fields = {"order": p, "q1d": int(q1d), "ne": int(ne), "nd_dofs": int(nd.ndofs), "rt_dofs": int(rt.ndofs), "gpu": name}
    for flux, smooth, config in (("rt", "nd", "curl_flux"), ("nd", "rt", "grad_flux")):
        arms = {
            "dense": capi.FluxEstimator(ctx, geom, dense[flux], dense[smooth], C, Cd, Cs, M[smooth], tol=1e-10, max_it=2000),
            "sum_factorised": capi.FluxEstimator.hex(ctx, geom, tens[flux], tens[smooth], C, Cd, Cs, M[smooth], tol=1e-10, max_it=2000),
        }
        y = torch.empty(n[smooth], dtype=torch.float64, device="cuda")
        est = torch.zeros(ne, dtype=torch.float64, device="cuda")
        out_f, out_i, ms_f, ms_i = {}, {}, {a: [] for a in arms}, {a: [] for a in arms}
        for a, E in arms.items():  # warm-up and outputs
            E.flux_mult(x[flux], y)
            est.zero_()
            E.integrate(x[flux], x[smooth], est)
            torch.cuda.synchronize()
            E.flux_mult(x[flux], y)
            out_f[a] = y.cpu().numpy().copy()
            est.zero_()
            E.integrate(x[flux], x[smooth], est)
            out_i[a] = est.cpu().numpy().copy()
        for _ in range(rounds):  # alternate the arms
            for a, E in arms.items():
                ms_f[a].append(time_calls(lambda: E.flux_mult(x[flux], y), flush, reps, torch))
                ms_i[a].append(time_calls(lambda: E.integrate(x[flux], x[smooth], est), flush, reps, torch))
        qbytes = 80 * Q * ne
        for a in arms:
            tabs = 8 * (interp[flux].size + interp[smooth].size) if a == "dense" else 0
            for what, ms, out, nb in (
                ("flux_mult", ms_f, out_f, 8 * (n[flux] + n[smooth]) + 4 * ne * (Pe[flux] + Pe[smooth]) + qbytes + 80 * ne + tabs),
                ("integrate", ms_i, out_i, 8 * (n[flux] + n[smooth]) + 4 * ne * (Pe[flux] + Pe[smooth]) + qbytes + 144 * ne + 16 * ne + tabs),
            ):
                m = float(np.median(ms[a]))
                ref = out["sum_factorised"]
                print(json.dumps({"bench": what, "config": config, "direction": f"{flux}->{smooth}" if what == "flux_mult" else None,
                                  "arm": a, **common_fields, "ms": round(m, 4), "ms_rounds": [round(v, 4) for v in ms[a]],
                                  "bytes": int(nb), "frac_of_3.35TB/s": round(nb / (m * 1e-3) / HBM, 3),
                                  "rel_diff_vs_sum_factorised": float(np.linalg.norm(out[a] - ref) / np.linalg.norm(ref)),
                                  "speedup_of_sum_factorised": round(m / float(np.median(ms["sum_factorised"])), 3)}), flush=True)
        if skip_indicator:
            continue
        for E in arms.values():
            ops, P = levels(ctx, mesh, prob.topo, smooth, nd if smooth == "nd" else rt, mop if smooth == "nd" else rop, M[smooth], q1d, orders)
            E.set_multigrid(ops, P, coarse_type=1, coarse_tol=1e-8, coarse_max_it=2000)
            E._bench_levels = (ops, P)
        ts, outs = {a: [] for a in arms}, {}
        for a, E in arms.items():
            E.indicator(x[flux], None, 0.0, est)  # warm-up
            torch.cuda.synchronize()
            outs[a] = est.cpu().numpy().copy()
        for _ in range(rounds):
            for a, E in arms.items():
                flush.zero_()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                E.indicator(x[flux], None, 0.0, est)
                torch.cuda.synchronize()
                ts[a].append(1e3 * (time.perf_counter() - t0))
        for a, E in arms.items():
            st = E.stats()
            m = float(np.median(ts[a]))
            print(json.dumps({"bench": "indicator", "config": config, "arm": a, **common_fields, "levels": orders, "iterations": st["its"],
                              "converged": st["converged"], "ms": round(m, 3), "ms_rounds": [round(v, 3) for v in ts[a]],
                              "rel_diff_vs_sum_factorised": float(np.linalg.norm(outs[a] - outs["sum_factorised"]) /
                                                                  np.linalg.norm(outs["sum_factorised"])),
                              "speedup_of_sum_factorised": round(m / float(np.median(ts["sum_factorised"])), 3)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--orders", type=int, nargs="+", default=[2, 3, 4, 5, 6])
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-indicator", action="store_true")
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "flux_hex_bench.py measures on the GPU; there is no CPU path"
    ctx = capi.Ctx(0)
    capi.set_stream(ctx)
    name = card()
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")  # larger than the 50 MB L2
    for p in args.orders:
        bench_order(ctx, p, args.reps, args.rounds, flush, name, torch, args.skip_indicator)


if __name__ == "__main__":
    main()

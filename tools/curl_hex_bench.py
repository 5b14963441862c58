#!/usr/bin/env python
"""Discrete curl ND_p -> RT_{p-1} on hexahedra, three routes alternated in one process at about 2M ND dofs per order on a box mesh:

  curl_hex  the sum-factorised curl kernel (b2p_interp_create_curl_hex, curl_hex_kernel): one launch per apply
  kron2     the same curl as two b2p_interp_create Kronecker handles, one per term of RT_c = D_a u_b - D_b u_a, applied one after
            the other (assemble.curl_kron_terms)
  dense     b2p_interp_create_dense with the element matrix hexspace.discrete_curl_matrix (p <= 4: larger elements are refused)

For Mult and MultTranspose: ms per call (CUDA events around each apply, L2 flushed before it, median over the rounds of the
per-round means; the arms alternate within each round), algorithmic bytes per call and their fraction of 3.35 TB/s, and the largest
difference between the arms' outputs on the same seeded input. Algorithmic bytes of one handle: a 4-byte index per element dof of
both restrictions, the input once and the output read and written once per unique dof (8 + 16 bytes), and the 8-byte 1/multiplicity
of the RT space; kron2 moves that twice, dense adds its matrix once.

Prints one JSON line per measurement with the card's name, power limit and max SM clock read in the same run.
  python tools/curl_hex_bench.py [--orders 1 2 3 4 5 6] [--reps 20] [--rounds 5] [--target 2e6]
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

from palace_b200 import capi  # noqa: E402
from palace_b200.host import assemble as asm  # noqa: E402
from palace_b200.host import hexmesh as hm  # noqa: E402
from palace_b200.host import hexspace as hs  # noqa: E402

HBM = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def box_side(p, target):
    """elements per side for about `target` ND dofs (3 p (p + 1)^2 per element, about 3 p^3 once shared dofs are counted once)"""
    return max(2, int(round((target / (3 * p ** 3)) ** (1.0 / 3.0))))


def handle_bytes(ne, P_nd, P_rt, n_in, n_out, rt_lsize):
    return 4 * ne * (P_nd + P_rt) + 8 * n_in + 16 * n_out + 8 * rt_lsize


def time_apply(its, x, y, transpose, flush, reps, torch):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        flush.zero_()
        a.record()
        for it in its:
            it.apply_add(x, y, transpose=transpose)
        b.record()
    torch.cuda.synchronize()
    return float(np.mean([a.elapsed_time(b) for a, b in ev]))


def bench_order(ctx, p, args, flush, name, torch):
    n1 = box_side(p, args.target)
    mesh = hm.box_mesh((n1, n1, n1), (1.0, 1.0, 1.0), n_attr=1)
    topo = hs.build_topology(mesh)
    nd, rt = hs.build_nd_space(mesh, topo, p), hs.build_rt_space(mesh, topo, p)
    snd, srt = asm.space_dict(nd), asm.space_dict(rt)
    arms = {"curl_hex": [capi.Interp.curl_hex(ctx, snd, srt, p)],
            "kron2": [capi.Interp(ctx, snd, srt, t) for t in asm.curl_kron_terms(p)]}
    Cl = hs.discrete_curl_matrix(p)
    if p <= 4:
        arms["dense"] = [capi.Interp.dense(ctx, Cl, nd.lex_gid, nd.ndofs, rt.lex_gid, rt.ndofs, in_orient=nd.lex_sign, out_orient=rt.lex_sign)]
    ne = mesh.ne
    for transpose in (False, True):
        n_in, n_out = (rt.ndofs, nd.ndofs) if transpose else (nd.ndofs, rt.ndofs)
        x = torch.from_numpy(np.random.default_rng(2024 + p).standard_normal(n_in)).cuda()
        y = torch.zeros(n_out, dtype=torch.float64, device="cuda")
        out, ms = {}, {a: [] for a in arms}
        for a, its in arms.items():  # warm-up (module load, first launches) and the outputs compared
            y.zero_()
            for it in its:
                it.apply_add(x, y, transpose=transpose)
            torch.cuda.synchronize()
            out[a] = y.cpu().numpy()
        for _ in range(args.rounds):
            for a, its in arms.items():
                ms[a].append(time_apply(its, x, y, transpose, flush, args.reps, torch))
        one = handle_bytes(ne, nd.P, rt.P, n_in, n_out, rt.ndofs)
        nbytes = {"curl_hex": one, "kron2": 2 * one, "dense": one + 8 * Cl.size}
        ref = out["curl_hex"]
        max_diff = max(float(np.abs(out[a] - ref).max()) for a in arms)
        m_kron = float(np.median(ms["kron2"]))
        for a in arms:
            m = float(np.median(ms[a]))
            print(json.dumps({"bench": "curl_hex", "order": p, "direction": "MultTranspose" if transpose else "Mult", "arm": a,
                              "ne": int(ne), "nd_dofs": int(nd.ndofs), "rt_dofs": int(rt.ndofs), "ms_per_call": round(m, 4),
                              "ms_rounds": [round(v, 4) for v in ms[a]], "bytes_per_call": int(nbytes[a]),
                              "frac_of_3.35TB/s": round(nbytes[a] / (m * 1e-3) / HBM, 3),
                              "rel_diff_vs_curl_hex": float(np.linalg.norm(out[a] - ref) / np.linalg.norm(ref)),
                              "max_abs_diff_between_arms": max_diff, "kron2_ms_over_this": round(m_kron / m, 3), "gpu": name}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--orders", type=int, nargs="+", default=[1, 2, 3, 4, 5, 6])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--target", type=float, default=2.0e6, help="ND dofs per order")
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "curl_hex_bench.py measures on the GPU; there is no CPU path"
    ctx = capi.Ctx(0)
    capi.set_stream(ctx)
    name = card()
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")  # larger than the 50 MB L2
    for p in args.orders:
        bench_order(ctx, p, args, flush, name, torch)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Complex Floquet matvec on a z-periodic hex box: y = (K_r + i K_i - sigma M) x with
K_r = curl-curl + mass([k x]^T [k x]) and K_i = weak curl + mixed curl (unit materials, k = (0, 0, kz)).

Three ways to run the same operator, alternated in one process:
  dense   hexahedra through dense interp / curl tables (b2p_op_create_dense), one real apply per term and part (dense sums
          do not take the mixed kinds)
  terms   sum-factorised operators, one real apply per term and part (B2P_COMPLEX_FUSED=0)
  block   sum-factorised S_re / S_im block sums (the default ComplexParOperator path)

Prints one JSON line per (order, arm): ms per complex matvec (CUDA events, after warm-up), GDoF/s, algorithmic bytes per
matvec (b2p_op_algorithmic_bytes of the real applies one matvec launches; an approximation for the block arm, see
bytes_per_matvec), the max relative difference of the arm's
output to the block arm's on the same seeded x, and the card name and power limit read in the same run.

  python tools/floquet_hex_bench.py [--orders 3 6] [--reps 20] [--rounds 3]
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
from palace_b200.host import coeff as cf  # noqa: E402
from palace_b200.host import hexmesh as hm  # noqa: E402
from tests import common  # noqa: E402

BOX = {2: 43, 3: 29, 6: 15}  # elements per side of the z-periodic box: 1.94M ND dofs at p = 2, 2.01M at p = 3, 2.22M at p = 6


def terms(kz, sigma):
    kx = np.array([[0.0, -kz, 0.0], [kz, 0.0, 0.0], [0.0, 0.0, 0.0]])
    am = np.array([0])
    one = cf.coeff_ctx(a=1.0)
    t = [(O.CURLCURL, one, 1.0), (O.ND_MASS, cf.coeff_ctx(am, (kx.T @ kx)[None]), 1.0),
         (O.ND_WEAKCURL, cf.coeff_ctx(am, kx[None], a=-1.0), 1j), (O.ND_MIXEDCURL, cf.coeff_ctx(am, kx[None], transpose=True), 1j),
         (O.ND_MASS, one, -sigma)]
    return t


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def build(ctx, prob, arm, t):
    nd, p = prob.nd, prob.p
    if arm == "dense":
        geom = capi.Geom.general(ctx, prob.qdata_ref)
        interp, curl, _ = O.nd_hex_tables(p, prob.q1d)
        idx, ori = nd.native_restriction()
        ops = [capi.Op.create_dense(ctx, geom, k, nd.ndofs, idx, ori, interp, curl, b) for k, b, _ in t]
    else:
        geom = common.gpu_geom(ctx, prob)
        ops = [common.gpu_op(ctx, geom, prob, k, b) for k, b, _ in t]
    os.environ["B2P_COMPLEX_FUSED"] = "0" if arm == "terms" else "1"
    A = capi.ComplexOperator.par(ctx, nd.ndofs, nd.ndofs, ops, [c for _, _, c in t], nd.ess_dofs, diag_policy=1)
    return prob, ops, A


def time_arm(A, xr, xi, yr, yi, reps, torch):
    A.mult(xr, xi, yr, yi)  # warm-up: module load, first launches
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        A.mult(xr, xi, yr, yi)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def bytes_per_matvec(arm, ops, t):
    """Algorithmic bytes of the real applies one complex matvec launches. For the block arm this is an APPROXIMATION: each of
    S_re and S_im is counted as the largest per-term byte count (a mixed term's, 288-byte coefficient block), which is the byte
    model of one block operator on the same space."""
    n_re = sum(1 for _, _, c in t if complex(c).real != 0.0)
    n_im = sum(1 for _, _, c in t if complex(c).imag != 0.0)
    if arm != "block":  # term by term (dense sums do not take the mixed kinds)
        return sum(2 * ((complex(c).real != 0.0) + (complex(c).imag != 0.0)) * o.algorithmic_bytes() for o, (_, _, c) in zip(ops, t))
    # S_re and S_im, each applied to both parts; each is modelled as one operator of the block form (the mixed terms' model)
    per = max(o.algorithmic_bytes() for o in ops)
    return 2 * ((n_re > 0) + (n_im > 0)) * per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--orders", type=int, nargs="+", default=[3, 6])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kz", type=float, default=0.4)
    ap.add_argument("--sigma", type=float, default=-1.0)
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "floquet_hex_bench.py measures on the GPU; there is no CPU path"
    ctx = capi.Ctx(0)
    capi.set_stream(ctx)
    name = card()
    t = terms(args.kz, args.sigma)
    for p in args.orders:
        n1 = BOX[p]
        prob = common.problem_on_mesh(hm.box_mesh((n1, n1, n1), (1.0, 1.0, 1.0), periodic_z=True), p=p, mesh_order=1)
        arms = {arm: build(ctx, prob, arm, t) for arm in ("dense", "terms", "block")}
        n = arms["block"][0].nd.ndofs
        rng = np.random.default_rng(2024)
        x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        xr, xi = torch.from_numpy(x.real.copy()).cuda(), torch.from_numpy(x.imag.copy()).cuda()
        out, ms = {}, {a: [] for a in arms}
        for arm, (_, _, A) in arms.items():
            yr, yi = torch.empty_like(xr), torch.empty_like(xi)
            A.mult(xr, xi, yr, yi)
            torch.cuda.synchronize()
            out[arm] = yr.cpu().numpy() + 1j * yi.cpu().numpy()
        for _ in range(args.rounds):  # alternate the arms
            for arm, (_, _, A) in arms.items():
                yr, yi = torch.empty_like(xr), torch.empty_like(xi)
                ms[arm].append(time_arm(A, xr, xi, yr, yi, args.reps, torch))
        ref = out["block"]
        for arm, (_, ops, _) in arms.items():
            m = float(np.median(ms[arm]))
            print(json.dumps({"order": p, "arm": arm, "ndofs": int(n), "ne": int(arms[arm][0].mesh.ne), "ms_per_matvec": round(m, 4),
                              "ms_all": [round(v, 4) for v in ms[arm]], "gdof_per_s": round(n / (m * 1e-3) / 1e9, 3),
                              "bytes_per_matvec": int(bytes_per_matvec(arm, ops, t)),
                              "max_rel_diff_vs_block": float(np.abs(out[arm] - ref).max() / np.abs(ref).max()),
                              "gpu": name}), flush=True)
        del arms
    ctx.close()


if __name__ == "__main__":
    main()

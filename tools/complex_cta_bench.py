#!/usr/bin/env python
"""Complex matvec on the CTA-per-batch kernel (nd_hex_apply7_kernel<..., CPLX>, one pass over the geometry for every term and
both parts) against the routes it replaces, alternated in one process at about 2M complex dofs:

  symmetric  K + lossy M + conductivity term (the sum of tools/zfused_bench.py) at p = 4, 5, 6
             terms     one real apply per term and part (B2P_COMPLEX_FUSED=0)
             two_sums  b2p_coperator_wrap of two fused b2p_operator_par (the real and the imaginary coefficient sums)
             one_pass  the default b2p_coperator_par route
  floquet    the Floquet block operator on the z-periodic box (tools/floquet_hex_bench.py) at p = 2 ... 6
             two_sums  as above (two block operators, 4 applies)
             one_pass  the default b2p_coperator_par route

Prints one JSON line per (workload, order, arm): ms per complex matvec (CUDA events around each matvec, L2 flushed before it,
median over the rounds of the per-round means), algorithmic bytes per matvec (DESIGN 3: x and y per unique dof, 4-byte index per
element dof, 80 bytes of q-data per point, the coefficient blocks), their fraction of 3.35 TB/s, the relative difference to the
one-pass output on the same seeded x, and the card's name, power limit and max SM clock read in the same run.
  python tools/complex_cta_bench.py [--workloads symmetric floquet] [--orders 4 5 6] [--reps 20] [--rounds 5]
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

# elements per side (about 3 p^3 n^3 ND dofs): 1.94M at p = 2, 2.01M at 3, 2.04M at 4, 1.84M at 5, 2.22M at 6
BOX = {2: 43, 3: 29, 4: 22, 5: 17, 6: 15}
HBM = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def terms(workload, kz=0.4, sigma=-1.0):
    """(kind, coefficient context, complex coefficient) of each term."""
    one = cf.coeff_ctx(a=1.0)
    if workload == "symmetric":
        return [(O.CURLCURL, one, 1.0 + 0.0j), (O.ND_MASS, one, -9.0 * (1 - 0.05j)), (O.ND_MASS, cf.coeff_ctx(a=0.3), 0.7j)]
    kx = np.array([[0.0, -kz, 0.0], [kz, 0.0, 0.0], [0.0, 0.0, 0.0]])
    am = np.array([0])
    return [(O.CURLCURL, one, 1.0), (O.ND_MASS, cf.coeff_ctx(am, (kx.T @ kx)[None]), 1.0),
            (O.ND_WEAKCURL, cf.coeff_ctx(am, kx[None], a=-1.0), 1j), (O.ND_MIXEDCURL, cf.coeff_ctx(am, kx[None], transpose=True), 1j),
            (O.ND_MASS, one, -sigma)]


def build(ctx, prob, t, arm):
    nd = prob.nd
    geom = common.gpu_geom(ctx, prob)
    ops = [common.gpu_op(ctx, geom, prob, k, b) for k, b, _ in t]
    c = [complex(v) for _, _, v in t]
    if arm == "two_sums":
        Ar = capi.Operator.par(ctx, nd.ndofs, nd.ndofs, ops, [v.real for v in c], nd.ess_dofs, diag_policy=1)
        Ai = capi.Operator.par(ctx, nd.ndofs, nd.ndofs, ops, [v.imag for v in c], nd.ess_dofs, diag_policy=0)
        assert Ar.is_fused() and Ai.is_fused()
        A = capi.ComplexOperator.wrap(ctx, Ar, Ai)
        A._keep += [ops]
        return A, ops
    os.environ["B2P_COMPLEX_FUSED"] = "0" if arm == "terms" else "1"
    A = capi.ComplexOperator.par(ctx, nd.ndofs, nd.ndofs, ops, c, nd.ess_dofs, diag_policy=1)
    assert A.fused_path() == (0 if arm == "terms" else 3), (arm, A.fused_path())
    return A, ops


def bytes_per_matvec(arm, ops, t):
    """Algorithmic bytes of the real applies one complex matvec launches (b2p_op_algorithmic_bytes). A fused real sum is counted as
    its largest term (the block form's 288-byte coefficient block when it holds a mixed term)."""
    c = [complex(v) for _, _, v in t]
    if arm == "terms":
        return sum(2 * ((v.real != 0) + (v.imag != 0)) * op.algorithmic_bytes() for op, v in zip(ops, c))
    n_re, n_im = any(v.real != 0 for v in c), any(v.imag != 0 for v in c)
    return 2 * (n_re + n_im) * max(op.algorithmic_bytes() for op in ops)


def one_pass_bytes(prob, block):
    """Both parts of x read and of y written once, the restriction and q-data streamed once, the complex coefficient block: 288
    bytes per element for the symmetric kinds, two 288-byte blocks for block sums."""
    u = 3 * prob.p * (prob.p + 1) ** 2
    ps = (u + 3) & ~3
    return 32 * prob.nd.ndofs + prob.mesh.ne * (4 * ps + 80 * prob.q1d ** 3 + (576 if block else 288))


def time_arm(A, xr, xi, yr, yi, flush, reps, torch):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        flush.zero_()
        a.record()
        A.mult(xr, xi, yr, yi)
        b.record()
    torch.cuda.synchronize()
    return float(np.mean([a.elapsed_time(b) for a, b in ev]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["symmetric", "floquet"])
    ap.add_argument("--orders", type=int, nargs="+", default=None)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "complex_cta_bench.py measures on the GPU; there is no CPU path"
    ctx = capi.Ctx(0)
    capi.set_stream(ctx)
    name = card()
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")  # larger than the 50 MB L2
    for wl in args.workloads:
        block = wl == "floquet"
        orders = args.orders or ([2, 3, 4, 5, 6] if block else [4, 5, 6])
        arm_names = ["two_sums", "one_pass"] if block else ["terms", "two_sums", "one_pass"]
        t = terms(wl)
        for p in orders:
            if not block and p < 4:
                continue
            n1 = BOX[p]
            mesh = hm.box_mesh((n1, n1, n1), (1.0, 1.0, 1.0), periodic_z=block)
            prob = common.problem_on_mesh(mesh, p=p, mesh_order=1)
            arms = {a: build(ctx, prob, t, a) for a in arm_names}
            n = prob.nd.ndofs
            rng = np.random.default_rng(2024)
            x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
            xr, xi = torch.from_numpy(x.real.copy()).cuda(), torch.from_numpy(x.imag.copy()).cuda()
            yr, yi = torch.empty_like(xr), torch.empty_like(xr)
            out, ms = {}, {a: [] for a in arms}
            for a, (A, _) in arms.items():
                A.mult(xr, xi, yr, yi)  # warm-up: module load, first launches
                torch.cuda.synchronize()
                out[a] = yr.cpu().numpy() + 1j * yi.cpu().numpy()
            for _ in range(args.rounds):  # alternate the arms
                for a, (A, _) in arms.items():
                    ms[a].append(time_arm(A, xr, xi, yr, yi, flush, args.reps, torch))
            ref = out["one_pass"]
            for a, (A, ops) in arms.items():
                m = float(np.median(ms[a]))
                nb = one_pass_bytes(prob, block) if a == "one_pass" else bytes_per_matvec(a, ops, t)
                print(json.dumps({"workload": wl, "order": p, "arm": a, "ndofs": int(n), "ne": int(prob.mesh.ne),
                                  "ms_per_matvec": round(m, 4), "ms_rounds": [round(v, 4) for v in ms[a]],
                                  "bytes_per_matvec": int(nb), "frac_of_3.35TB/s": round(nb / (m * 1e-3) / HBM, 3),
                                  "rel_diff_vs_one_pass": float(np.linalg.norm(out[a] - ref) / np.linalg.norm(ref)),
                                  "speedup_of_one_pass": round(m / float(np.median(ms["one_pass"])), 3), "gpu": name}), flush=True)
            del arms


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""A/B of the geometry source of nd_hex_apply6_kernel on bench.py's workload: the same ND p = 3 curl-curl + mass ParOperator::Mult
on the same trilinear box, once on Geom.hex (the kernel evaluates the geometry from the element vertices) and once on
Geom.from_qdata of that geometry's q-data (the kernel streams the stored per-point q-data). Both operators live in one process and
are timed in alternation, round after round, with the L2 flushed (256 MiB write) before every step and CUDA events around it.
Prints one JSON line per round and a summary line: us per Mult and per element-kernel launch of each arm, the largest relative
difference of the two outputs on bench.py's x, and the GPU name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, plim = [v.strip() for v in out.split(",")]
        return name, plim
    except Exception as exc:
        return f"unknown ({type(exc).__name__})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=29)
    ap.add_argument("--order", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200, help="timed Mults per arm and round")
    ap.add_argument("--kernel-steps", type=int, default=50, help="timed element-kernel launches per arm and round")
    ap.add_argument("--coefficient", default="iso", choices=["iso", "matrix4"])
    ap.add_argument("--warp", type=float, default=0.0)
    args = ap.parse_args()
    import torch

    from palace_b200 import capi

    assert torch.cuda.is_available(), "geom_nodes_ab.py needs a GPU"
    ctx = capi.Ctx(0)
    capi.set_stream(ctx)
    stream = torch.cuda.current_stream()
    prob = bench.build_problem((args.n,) * 3, args.order, args.warp, coefficient=args.coefficient)
    nd, p, q1d, t = prob["nd"], prob["p"], prob["q1d"], prob["tabs"]
    geom_nodes = capi.Geom.hex(ctx, prob["xe"], prob["mesh"].attr, prob["mesh_order"], q1d, prob["nB"], prob["nG"], t.qw)
    geom_stored = capi.Geom.from_qdata(ctx, geom_nodes.qdata(), q1d)
    idx, ori = nd.native_restriction()
    n = nd.ndofs
    arms = {}
    for name, g in (("nodes", geom_nodes), ("qdata", geom_stored)):
        op = capi.Op.create(ctx, g, capi.CURLCURL_MASS, p, n, idx, ori, nd.dof_map, t.Bo, t.Bc, t.Gc, prob["blob"])
        arms[name] = (op, capi.Operator.par(ctx, n, n, [op], None, None, diag_policy=1))
    xd = torch.from_numpy(np.random.default_rng(1).random(n)).cuda()  # bench.py's x (seed 1 + rank 0)
    yd = torch.empty_like(xd)
    yl = torch.zeros(n, dtype=torch.float64, device="cuda")
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")

    outs, routes = {}, {}
    for name, (op, A) in arms.items():
        for _ in range(10):
            A.mult(xd, yd)
        torch.cuda.synchronize()
        outs[name] = yd.cpu().numpy()
        op.apply_add(xd, yl)
        r = capi.last_launch(ctx)
        routes[name] = f'{r["kernel"]}/{r["geom"]}'
    diff = float(np.abs(outs["nodes"] - outs["qdata"]).max() / np.abs(outs["qdata"]).max())

    def timed(fn, steps):
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for a, b in evs:
            flush.zero_()
            a.record(stream)
            fn()
            b.record(stream)
        torch.cuda.synchronize()
        return 1e3 * float(np.mean([a.elapsed_time(b) for a, b in evs]))

    mult = {k: [] for k in arms}
    kern = {k: [] for k in arms}
    for rnd in range(args.rounds):
        for name, (op, A) in arms.items():
            mult[name].append(timed(lambda: A.mult(xd, yd), args.steps))
            kern[name].append(timed(lambda: op.apply_add(xd, yl), args.kernel_steps))
        print(json.dumps({"round": rnd, **{f"{k}_us_per_mult": round(mult[k][-1], 2) for k in arms},
                          **{f"{k}_us_per_kernel": round(kern[k][-1], 2) for k in arms}}), flush=True)
    gname, plim = gpu_info()
    summary = {
        "workload": f"ND p={p} curl-curl+mass ParOperator Mult, {args.n}^3 trilinear box, {n} dofs, {args.coefficient} coefficient, "
                    f"L2 flushed between steps",
        "routes": routes,
        "us_per_mult": {k: {"min": round(min(v), 2), "max": round(max(v), 2), "mean": round(float(np.mean(v)), 2)} for k, v in mult.items()},
        "us_per_kernel": {k: {"min": round(min(v), 2), "max": round(max(v), 2), "mean": round(float(np.mean(v)), 2)} for k, v in kern.items()},
        "mult_gain": round(1.0 - float(np.mean(mult["nodes"])) / float(np.mean(mult["qdata"])), 4),
        "algorithmic_bytes": {k: arms[k][0].algorithmic_bytes() for k in arms},
        "max_rel_diff_nodes_vs_qdata": diff,
        "rounds": args.rounds, "steps": args.steps, "kernel_steps": args.kernel_steps,
        "gpu": gname, "power_limit": plim,
    }
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()

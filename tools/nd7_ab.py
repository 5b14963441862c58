#!/usr/bin/env python
"""A/B of the sum-factorised ND hexahedron kernels on one GPU: nd_hex_apply4_kernel (warp per element) against
nd_hex_apply7_kernel (CTA per element batch) in its launch shapes (B2P_ND7_CFG), curl-curl + mass, isotropic
coefficient, L2 flushed between launches. One JSON line per (order, variant): kernel time, GDoF/s, fraction of the
measured HBM peak on bench.py's byte model, and the largest relative difference to nd_hex_apply4_kernel's result."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--orders", default="4,5,6")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--configs", default="2:317c,318g,318c,319c,724c;3:217c,218g,218c,219c,324c,424c;4:118g,118c,542c;5:232g,232c,341c;6:123g,123c,122c",
                    help="B2P_ND7_CFG values per order: <elements per batch><warps per component><CTAs per SM><d|g|c>")
    ap.add_argument("--skip-round1", action="store_true")
    ap.add_argument("--default-arm", action="store_true",
                    help="also time the call without kernel flags (the kernel B2P_ND_KERNEL selects, or the default)")
    ap.add_argument("--warp", type=float, default=0.0)
    ap.add_argument("--coefficient", default="iso")
    args = ap.parse_args()
    import torch

    from palace_b200 import capi

    ctx = capi.Ctx(0)
    capi.set_stream(ctx)
    stream = torch.cuda.current_stream()
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    peak, _ = bench.measured_peak_gbs()
    sizes = {2: 40, 3: 29, 4: 23, 5: 18, 6: 15}
    for p in [int(v) for v in args.orders.split(",")]:
        n = sizes[p]
        prob = bench.build_problem((n, n, n), p, args.warp, coefficient=args.coefficient)
        nd = prob["nd"]
        geom = capi.Geom.hex(ctx, prob["xe"], prob["mesh"].attr, prob["mesh_order"], prob["q1d"], prob["nB"], prob["nG"], prob["tabs"].qw)
        idx, ori = nd.native_restriction()
        t = prob["tabs"]
        op = capi.Op.create(ctx, geom, capi.CURLCURL_MASS, p, nd.ndofs, idx, ori, nd.dof_map, t.Bo, t.Bc, t.Gc, prob["blob"], assemble=False)
        x = torch.from_numpy(np.random.default_rng(5).random(nd.ndofs)).cuda()
        y = torch.zeros_like(x)
        abytes = op.algorithmic_bytes()
        y_ref = None

        def run(name, **kw):
            nonlocal y_ref
            for _ in range(3):
                y.zero_()
                op.apply_add_ex(1.0, x, y, **kw)
            torch.cuda.synchronize()
            yy = y.clone()
            if y_ref is None:
                y_ref = yy
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.reps)]
            for a, b in evs:
                y.zero_()
                flush.zero_()
                a.record(stream)
                op.apply_add_ex(1.0, x, y, **kw)
                b.record(stream)
            torch.cuda.synchronize()
            ms = np.array([a.elapsed_time(b) for a, b in evs])
            k_ms = float(ms.mean())
            diff = float((yy - y_ref).abs().max() / y_ref.abs().max())
            print(json.dumps({"order": p, "elements": int(prob["mesh"].ne), "dofs": int(nd.ndofs), "variant": name, "kernel_ms": k_ms,
                              "kernel_ms_min": float(ms.min()), "GDoF_per_s": nd.ndofs / (k_ms * 1e-3) / 1e9,
                              "roofline_frac": abytes / (k_ms * 1e-3) / 1e9 / peak, "rel_diff_to_nd_hex_apply4": diff}), flush=True)

        if not args.skip_round1:
            run("nd_hex_apply4_kernel", round1_kernel=True)
        if args.default_arm:
            run("default B2P_ND_KERNEL=" + os.environ.get("B2P_ND_KERNEL", "0"))
        cfgs = dict(part.split(":") for part in args.configs.split(";"))
        for cfg in cfgs.get(str(p), "").split(","):
            if not cfg:
                continue
            os.environ["B2P_ND7_CFG"] = cfg
            try:
                run("nd_hex_apply7_kernel cfg=" + cfg, cta_kernel=True)
            except Exception as exc:  # (a shape that does not fit the SM)
                print(json.dumps({"order": p, "variant": "nd_hex_apply7_kernel cfg=" + cfg, "failed": str(exc)[:200]}), flush=True)
        os.environ.pop("B2P_ND7_CFG", None)
        del op, geom


if __name__ == "__main__":
    main()

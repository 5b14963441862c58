"""CPU check of the KERNEL SOURCES before any GPU time is spent: the `-m gpu` parity tests of the element
operators are re-run in a subprocess against tests/emu/libb2p_emu.so -- palace_b200/csrc compiled for the
SIMT-on-fibers emulation of tests/emu/cuda_emu.hpp (warps, barriers, shuffles, DMMA fragments, TMA + mbarrier
protocol, deferred cp.async). Test infrastructure only: this is not a GPU parity claim and no product path can
reach the emulation (B2P_EMU is defined only by tests/emu/Makefile; capi.py loads libb2p.so and nothing else)."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(files, order, extra=(), env=None):
    env = dict(os.environ, B2P_EMU_TESTS="1", B2P_EMU_ORDER=order, **(env or {}))
    cmd = [sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider", *extra, *files]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) > 0, tail
    return int(m.group(1))


def test_product_library_has_no_emulation_code():
    """The shipped library is built without B2P_EMU: no emulation symbol may appear in it."""
    lib = os.path.join(ROOT, "palace_b200", "libb2p.so")
    if not os.path.exists(lib):
        pytest.skip("libb2p.so not built")
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    assert "cuda_emu" not in out and "b2p_emu_switch" not in out


@pytest.mark.parametrize("order", ["fwd", "rev"])
def test_element_kernels_under_emulation(order):
    """Sum-factorised ND / H1 hex kernels (production, simple and half-warp variants), the dense DMMA operator,
    the tetrahedron path, the fused complex kernel, the kernel each hex apply is routed to: every parity test of these files must also hold on the emulated SIMT machine, for two
    different lane execution orders (a missing warp barrier shows up as stale data in at least one of them)."""
    n = _run(["tests/test_apply_gpu.py", "tests/test_dense_gpu.py", "tests/test_tet_gpu.py", "tests/test_zfused_gpu.py", "tests/test_zassemble_gpu.py", "tests/test_zbdr_gpu.py", "tests/test_zsolver_variants_gpu.py", "tests/test_zsum_gpu.py", "tests/test_zzhex_routes_gpu.py"], order)
    assert n >= 120


@pytest.mark.parametrize("order", ["fwd", "rev"])
def test_persistent_kernels_in_steady_state_under_emulation(order):
    """tests/test_zzsteady_state_gpu.py on ONE emulated SM: the meshes it sizes from the launch records stay small, and every
    warp or CTA of the persistent ND / H1 hex kernels still walks several element batches (ring slots reused, mbarrier parities
    flipped, next-batch prefetches), in both lane execution orders."""
    assert _run(["tests/test_zzsteady_state_gpu.py"], order, env={"B2P_EMU_SMS": "1"}) >= 97


def test_solver_layer_under_emulation():
    """Vector kernels, smoothers, interpolators, V-cycle and Krylov solvers: the whole device-resident loop of
    tests/test_solvers_gpu.py the divergence-free projection of tests/test_divfree_gpu.py and the flux error estimator of
    tests/test_zzflux_estimator_gpu.py on the emulated machine (reductions use two blocks per emulated SM)."""
    assert _run(["tests/test_solvers_gpu.py", "tests/test_divfree_gpu.py", "tests/test_zzflux_estimator_gpu.py"], "fwd") >= 34

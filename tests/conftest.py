import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (sm_90a; run with -m gpu)")
    if os.environ.get("B2P_EMU_TESTS") == "1":
        # pre-GPU validation: the same tests against the host-thread SIMT emulation build of the kernel sources
        from tests.emu import emu_mode

        emu_mode.enable()


def pytest_collection_modifyitems(config, items):
    # a wedged test must end the run instead of hanging it (pytest-timeout, when installed and no --timeout given)
    if config.pluginmanager.hasplugin("timeout") and not config.getoption("timeout", None):
        for item in items:
            if item.get_closest_marker("timeout") is None:
                item.add_marker(pytest.mark.timeout(1500))


@pytest.fixture(scope="session")
def b2p_ctx():
    from palace_b200 import capi

    ctx = capi.Ctx(0)
    yield ctx
    ctx.close()

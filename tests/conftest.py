import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "slow: long-running CPU test")


@pytest.fixture(scope="session")
def gpu_ctx():
    """Context on cuda:0 through the C ABI.  Fails loudly (no fallback) if the extension is missing."""
    from co_snarks_b200 import binding as B
    ctx = B.Context(0)
    yield ctx
    ctx.close()


@pytest.fixture(scope="session")
def emu_ctx():
    """Context on the CPU emulation build of the kernels (tests/emu) -- test infrastructure only."""
    from co_snarks_b200 import binding as B
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build_emu
    path = build_emu.build()
    ctx = B.Context(0, lib_path=path)
    yield ctx
    ctx.close()

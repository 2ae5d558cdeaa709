import ctypes
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with `pytest -m gpu`)")


@pytest.fixture(scope="session")
def orc():
    """tier-1 C oracle (oracle/c/ark_oracle.c) behind numpy helpers"""
    from oracle import loader
    loader.lib()
    return loader


@pytest.fixture(scope="session")
def emul_lib():
    """CPU kernel-logic emulator build of the library (tests/emul; NOT a product backend)"""
    from tests.emul import build as emul_build
    from distributed_plonk_b200._binding import bind
    # DP_TEST_EMUL_ASYNC=1 runs every emulator test on the asynchronous-stream build (streams are threads,
    # random delays): slower, used to hunt missing stream / event dependencies
    return bind(ctypes.CDLL(emul_build.build(async_streams=os.environ.get("DP_TEST_EMUL_ASYNC", "0") == "1")))


@pytest.fixture(scope="session")
def gpu_lib():
    """the real nvcc-built library; GPU tests fail (not skip) if it is missing.
    DP_TEST_DRY_RUN_ON_EMULATOR=1 (never set by the suite) hands a `-m gpu` test file the kernel-logic emulator instead,
    to check the test code itself on a box without a GPU (files that honour it shrink their sizes)."""
    if os.environ.get("DP_TEST_DRY_RUN_ON_EMULATOR", "0") == "1":
        from tests.emul import build as emul_build
        from distributed_plonk_b200._binding import bind
        return bind(ctypes.CDLL(emul_build.build()))
    import distributed_plonk_b200 as dp
    return dp.load()

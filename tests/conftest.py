import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _make(target):
    csrc = os.path.join(ROOT, "gnark_b200", "csrc")
    subprocess.check_call(["make", "-j", str(os.cpu_count() or 1), "-C", csrc, target])


@pytest.fixture(scope="session")
def hostemu():
    """CPU build of the device templates (PTX carry chains emulated) - test scaffolding."""
    import ctypes
    _make("../../tests/_build/libgb200_hostemu.so")
    return ctypes.CDLL(os.path.join(ROOT, "tests", "_build", "libgb200_hostemu.so"))


@pytest.fixture(scope="session")
def b200lib():
    """The product library (dlopen only; no CUDA call)."""
    path = os.path.join(ROOT, "gnark_b200", "lib", "libgnark_b200.so")
    if not os.path.exists(path):
        _make("../lib/libgnark_b200.so")
    from gnark_b200 import lib
    return lib.load()


@pytest.fixture(scope="session")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from gnark_b200 import lib
    lib.load()
    lib.init([0])
    return lib

import importlib
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

PKG_NAME = "comfyui-vrgamedevgirl_b200"
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with -m gpu)")


@pytest.fixture(scope="session")
def pkg():
    """The product package (directory name is not an identifier -> importlib)."""
    return importlib.import_module(PKG_NAME)


@pytest.fixture(scope="session")
def oracle():
    import vrgdg_oracle
    return vrgdg_oracle


@pytest.fixture(scope="session")
def hostcheck():
    """tests/hostcheck: the kernels' arithmetic header compiled for the host (test infrastructure)."""
    import ctypes
    d = os.path.join(ROOT, "tests", "hostcheck")
    so = os.path.join(d, "libhostcheck.so")
    src = os.path.join(d, "hostcheck.cpp")
    hdr = os.path.join(ROOT, PKG_NAME, "csrc", "vrgdg_math.cuh")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(hdr)):
        subprocess.run(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", src, "-o", so], check=True)
    return ctypes.CDLL(so)


@pytest.fixture(scope="session")
def cuda_device():
    """GPU tests must FAIL (not skip) when the box has no usable GPU or the library is missing."""
    import torch
    assert torch.cuda.is_available(), "pytest -m gpu needs a CUDA device"
    return torch.device("cuda", 0)

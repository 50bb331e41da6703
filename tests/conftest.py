import ctypes
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


def _build_if_missing(target, cmd, cwd):
    if not os.path.exists(target):
        subprocess.run(cmd, cwd=cwd, check=True, capture_output=True)
    return target


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (oracle/libkaspa_oracle.so): the CHECKER, never the thing under test."""
    path = _build_if_missing(os.path.join(ROOT, "oracle", "libkaspa_oracle.so"), ["make", "-C", os.path.join(ROOT, "oracle")], ROOT)
    lib = ctypes.CDLL(path)
    lib.ok_secp_init()
    return lib


@pytest.fixture(scope="session")
def gpu_ctx():
    import rusty_kaspa_b200 as rk
    ctx = rk.GpuContext(0)  # raises loudly if libkgv.so or the device is missing
    yield ctx
    ctx.close()


def oracle_schnorr_batch(lib, pk, msg, sig, threads=None):
    import numpy as np
    n = len(pk)
    st = np.zeros(n, dtype=np.uint8)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    lib.ok_schnorr_verify_batch(vp(pk), vp(msg), vp(sig), ctypes.c_size_t(n), vp(st), threads or min(32, os.cpu_count() or 1))
    return st


def oracle_ecdsa_batch(lib, pk, msg, sig, threads=None):
    import numpy as np
    n = len(pk)
    st = np.zeros(n, dtype=np.uint8)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    lib.ok_ecdsa_verify_batch(vp(pk), vp(msg), vp(sig), ctypes.c_size_t(n), vp(st), threads or min(32, os.cpu_count() or 1))
    return st

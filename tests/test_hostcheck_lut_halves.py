"""The split LUT cell evaluation (csrc/vrgdg_math.cuh: lut_half / lut_combine, lutp_half / lutp_combine; slot 4X + 2Y + Z) compiled
for the HOST with g++ and compared bit for bit with a whole-sector evaluation of the same corners on random tables and fractions
(tests/hostcheck/lut_halves.cpp).  The tile kernels' lane-pair gather evaluates one half per lane and combines on the owner lane, so
this equality is what makes its results identical to the per-lane gather."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostcheck", "lut_halves.cpp")


def _lib(tmp_path):
    so = str(tmp_path / "liblut_halves.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", so], check=True)
    lib = ctypes.CDLL(so)
    lib.lh_check.restype = ctypes.c_int64
    lib.lh_check.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int64)]
    return lib


def _check(lib, lut, f):
    lut = np.ascontiguousarray(lut, dtype=np.float32)
    f = np.ascontiguousarray(f, dtype=np.float32)
    checked = ctypes.c_int64(0)
    bad = lib.lh_check(lut.ctypes.data, lut.shape[0], f.ctypes.data, f.shape[0], ctypes.byref(checked))
    S = lut.shape[0]
    assert checked.value == S ** 3 * 3 * (16 + 6 * f.shape[0])
    return bad


def _fractions(rng, n):
    f = rng.random((n, 3), dtype=np.float32)
    f[:8] = [[0, 0, 0], [1, 1, 1], [0.5, 0.25, 0.75], [0, 1, 0], [1, 0, 1], [2.0 ** -24, 0.5, 1 - 2.0 ** -24], [0.1, 0.2, 0.3], [0.9, 0.8, 0.7]]
    return f


def test_lut_halves_match_whole_sector_on_random_tables(tmp_path):
    lib = _lib(tmp_path)
    rng = np.random.default_rng(20261015)
    f = _fractions(rng, 64)
    for S in (2, 5, 9):
        assert _check(lib, rng.random((S, S, S, 3), dtype=np.float32), f) == 0                    # a [0,1] table
    # values that leave [0,1] and lie far apart (1e3 next to 1e-30): coefficient differences are then not exact in double, so the
    # order in which the packer forms them (r, then g, then b) is visible; a constant channel has all-zero gradient coefficients
    S = 7
    wild = rng.choice(np.array([0.0, 1e-30, -1e-30, 1.0, 0.3, 1e3, -1e3], dtype=np.float32), (S, S, S, 3))
    wild[..., 1] = 0.25
    assert _check(lib, wild, f) == 0
    # a smooth table near identity (what a grading LUT looks like) at a shipped size
    S = 17
    ax = np.linspace(0, 1, S, dtype=np.float32)
    bb, gg, rr = np.meshgrid(ax, ax, ax, indexing="ij")
    smooth = np.stack([rr * 0.9 + 0.05 * gg, gg ** 1.2, 0.8 * bb + 0.1 * rr * gg], axis=-1)
    assert _check(lib, smooth, _fractions(rng, 16)) == 0

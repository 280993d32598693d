"""The fused restore kernel's matrix: the cases tests/test_gpu_restore_stream.py runs (k_restore against the resize -> blend
composition it replaces, and against the oracle), and a parser of what launch_restore and the ABI build, so that the CPU suite can
check that every (dtype, mode, channel count, store path) instantiation has a case (tests/test_restore_stream_cpu.py).  No GPU and
no torch needed here."""
import itertools
import re
from collections import namedtuple

import video_tools_matrix as vtm

MODES = vtm.RESIZE_MODES
FLOAT_DTYPES = vtm.FLOAT_DTYPES
CHANNELS = (3, 4)
# "stretch": the enhanced frame is resampled whole; "letterbox": the restore ROI of a letterboxed working frame
GEOMETRIES = {"stretch": ("Stretch to dimensions", (13, 17)), "letterbox": ("Fit with letterbox (preserve all)", (24, 24))}
# output widths: 27 takes the one-pixel-per-thread path, 32 the 16-byte path (a multiple of 16 / sizeof(T) pixels for every dtype)
WIDTHS = {"odd": 27, "aligned": 32}
FRAMES, HEIGHT = 3, 21
N_RESTORED = (0, 2, 3)                       # none, fewer than the originals, all of them
STRENGTHS = (0.0, 0.35, 1.0)

RestoreCase = namedtuple("RestoreCase", "mode dtype co ce geometry width")
CASES = [RestoreCase(*k) for k in itertools.product(MODES, FLOAT_DTYPES, CHANNELS, CHANNELS, GEOMETRIES, WIDTHS)]


def case_id(c):
    return "%s-%s-co%d-ce%d-%s-%s" % (c.mode, c.dtype, c.co, c.ce, c.geometry, c.width)


def store_path(c):
    """the path launch_restore takes for a case's frames (fresh torch allocations are 16-byte aligned)"""
    return "vec" if WIDTHS[c.width] % (16 // {"f32": 4, "f16": 2, "bf16": 2}[c.dtype]) == 0 else "scalar"


def kernel_of(c):
    return (c.dtype, c.mode, c.co, store_path(c))


def oracle_bar(c):
    """max |fused - oracle| (oracle.restore_batch + oracle.restore_blend on the up-cast input): the resize matrix's bars"""
    return vtm.resize_bar(vtm.ResizeCase(c.mode, c.dtype, c.co, "restore"))


def instantiated():
    """{(dtype, mode, Co, store path)} that launch_restore can run: its mode switch x launch_restore_m's (Co, VEC) calls x the
    dtypes the ABI dispatches to (float only) and VRGDG_INSTANTIATE builds"""
    src = vtm._read("vrgdg_resize.cuh")
    body = vtm._function_body(src, "template <typename T>\ncudaError_t launch_restore(")
    modes = set(m.lower() for m in re.findall(r"launch_restore_m<T, VRGDG_RESIZE_(\w+)>", body))
    assert "default: return launch_restore_m<T, VRGDG_RESIZE_AREA>" in body
    inner = vtm._function_body(src, "template <typename T, int MODE>\nstatic cudaError_t launch_restore_m(")
    paths = set((int(co), "vec" if v == "true" else "scalar") for co, v in re.findall(r"launch_restore_k<T, MODE, (\d), (true|false)>", inner))
    abi = vtm._abi_body("vrgdg_restore_blend")
    assert "dtype == VRGDG_U8BGR) return fail" in abi and "(Co != 3 && Co != 4)" in abi and "(Ce != 3 && Ce != 4)" in abi
    dts = set(vtm.CTYPE[t] for t in re.findall(r"RB\((\w+)\)", abi) if t in vtm.CTYPE) & vtm.instantiated_dtypes("VRGDG_INSTANTIATE")
    return {(dt, m, co, p) for dt, m, (co, p) in itertools.product(dts, modes, paths)}

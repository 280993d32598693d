"""The C-ABI library loads on a machine without a GPU and exports every symbol include/vrgdg_b200.h declares; the
ctypes table mirrors the header.  No compute calls here."""
import ctypes
import os
import re
import subprocess

import pytest

from conftest import PKG_NAME, ROOT

HEADER = os.path.join(ROOT, "include", "vrgdg_b200.h")


def declared_symbols():
    with open(HEADER, encoding="utf-8") as fh:
        text = fh.read()
    return sorted(set(re.findall(r"VRGDG_API\s+[\w\s\*]+?\b(vrgdg_\w+)\s*\(", text)))


def test_header_declares_the_expected_surface():
    names = declared_symbols()
    for must in ("vrgdg_lut3d_apply", "vrgdg_grain", "vrgdg_stencil3x3", "vrgdg_lab_moments", "vrgdg_colormatch_params",
                 "vrgdg_colormatch_apply", "vrgdg_chain_apply", "vrgdg_chain_lab_moments", "vrgdg_u8bgr_to_rgb", "vrgdg_rgb_to_u8bgr",
                 "vrgdg_version", "vrgdg_last_error"):
        assert must in names
    assert len(names) >= 18


def test_library_exports_every_declared_symbol(pkg):
    nv = pkg._native
    if not os.path.exists(nv.LIB_PATH):
        import importlib
        importlib.import_module(PKG_NAME + ".build").build()
    lib = ctypes.CDLL(nv.LIB_PATH)
    for name in declared_symbols():
        assert hasattr(lib, name), name
    assert sorted(nv.SIGNATURES) == declared_symbols()
    # exported dynamic symbols are exactly the ABI (everything else is hidden)
    out = subprocess.run(["nm", "-D", "--defined-only", nv.LIB_PATH], capture_output=True, text=True).stdout
    exported = sorted(l.split()[-1] for l in out.splitlines() if " T " in l and "vrgdg_" in l)
    assert exported == declared_symbols()


def test_version_and_error_channel_without_gpu(pkg):
    import torch
    nv = pkg._native
    lib = nv.load_library()
    assert lib.vrgdg_version() == 1
    assert lib.vrgdg_lab_moments_scratch_bytes(3) == 3 * 592 * 48
    if not torch.cuda.is_available():
        rc = lib.vrgdg_device_info(None, None, None)
        assert rc == nv.E_CUDA
        with pytest.raises(RuntimeError):
            nv.check(rc)
        # argument validation happens before any CUDA call
        rc = lib.vrgdg_stencil3x3(None, None, 1, 4, 4, 7, 1, 0.5, 0, None)
        assert rc == nv.E_INVALID and b"dtype" in lib.vrgdg_last_error()
        with pytest.raises(ValueError):
            nv.check(rc)


def test_sass_contains_tma_and_no_legacy_tensor_paths(pkg):
    """sm_90a only; the tile kernels use TMA (UTMALDG) + mbarrier (SYNCS); nothing routes through HMMA."""
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not installed")
    lst = subprocess.run([cuobjdump, "-lelf", pkg._native.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"\.(sm_\w+)\.cubin", lst))
    assert archs == {"sm_90a"}, archs


def test_header_is_plain_c_and_matches_the_ctypes_structs(pkg, tmp_path):
    """include/vrgdg_b200.h must compile as C99 on its own (the boundary is a C ABI, not C++), and the descriptor structs must have
    the size the ctypes mirrors in _native.py assume (a silent mismatch would shift every field after it)."""
    import ctypes
    import shutil
    import subprocess
    from conftest import ROOT
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    hdr = os.path.join(ROOT, "include", "vrgdg_b200.h")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-x", "c", hdr], check=True)
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include "vrgdg_b200.h"\nint main(void) { printf("%zu %zu %zu\\n", sizeof(vrgdg_chain_desc), '
                   'sizeof(vrgdg_adjust_desc), sizeof(vrgdg_resize_desc)); return 0; }\n')
    exe = tmp_path / "sizes"
    subprocess.run([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    sizes = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    nv = pkg._native
    assert sizes == [ctypes.sizeof(nv.ChainDesc), ctypes.sizeof(nv.AdjustDesc), ctypes.sizeof(nv.ResizeDesc)]


def test_argument_validation_of_the_widened_entry_points_needs_no_gpu(pkg):
    """resize / blend / Lanczos / adjust reject bad arguments with VRGDG_E_INVALID (-> ValueError) and a message naming the entry point,
    before any CUDA call (so this runs on the CPU-only build box too)."""
    import ctypes
    nv = pkg._native
    lib = nv.load_library()
    one = ctypes.c_void_p(16)                                     # a non-null, never dereferenced pointer
    rd = nv.ResizeDesc(2, 0, 0, 8, 8, 16, 16, 0, 0)
    cases = [
        (lambda: lib.vrgdg_resize(one, ctypes.c_void_p(32), 1, 8, 8, 3, 16, 16, 0, None, None), b"vrgdg_resize"),                    # null descriptor
        (lambda: lib.vrgdg_resize(one, ctypes.c_void_p(32), 1, 8, 8, 2, 16, 16, 0, ctypes.byref(rd), None), b"channels"),
        (lambda: lib.vrgdg_resize(one, ctypes.c_void_p(32), 1, 8, 8, 3, 16, 16, 3, ctypes.byref(rd), None), b"float dtype"),         # uint8 frames
        (lambda: lib.vrgdg_resize(one, ctypes.c_void_p(32), 1, 8, 8, 3, 16, 16, 0, ctypes.byref(nv.ResizeDesc(9, 0, 0, 8, 8, 16, 16, 0, 0)), None), b"mode"),
        (lambda: lib.vrgdg_resize(one, ctypes.c_void_p(32), 1, 8, 8, 3, 16, 16, 0, ctypes.byref(nv.ResizeDesc(2, 4, 0, 8, 8, 16, 16, 0, 0)), None), b"ROI"),
        (lambda: lib.vrgdg_resize(one, one, 1, 8, 8, 3, 16, 16, 0, ctypes.byref(rd), None), b"in-place"),
        (lambda: lib.vrgdg_blend(one, one, one, -1, 0, 0.5, 0.5, None), b"vrgdg_blend"),
        (lambda: lib.vrgdg_blend(None, one, one, 4, 0, 0.5, 0.5, None), b"null"),
        (lambda: lib.vrgdg_lanczos4_resize_u8(one, ctypes.c_void_p(32), 1, 8, 8, 16, 16, None, None, None, None, None, 0, None), b"null"),
        (lambda: lib.vrgdg_lanczos4_resize_u8(one, ctypes.c_void_p(32), 1, 0, 8, 16, 16, one, one, one, one, one, 1 << 20, None), b"empty source"),
        (lambda: lib.vrgdg_lanczos4_resize_u8(one, ctypes.c_void_p(32), 1, 8, 8, 16, 16, one, one, one, one, one, 4, None), b"scratch too small"),
        (lambda: lib.vrgdg_adjust(one, ctypes.c_void_p(32), 1, 8, 8, 0, None, None, None, None, 0, None), b"vrgdg_adjust"),
    ]
    for call, needle in cases:
        rc = call()
        assert rc == nv.E_INVALID and needle in lib.vrgdg_last_error(), (rc, needle, lib.vrgdg_last_error())
    # the message belongs to the LAST failing call on this thread
    assert b"vrgdg_adjust" in lib.vrgdg_last_error()
    rc = lib.vrgdg_blend(None, one, one, 4, 0, 0.5, 0.5, None)
    assert rc == nv.E_INVALID and b"vrgdg_blend" in lib.vrgdg_last_error()
    with pytest.raises(ValueError):
        nv.check(rc)
    # zero-sized work is a successful no-op before any CUDA call
    assert lib.vrgdg_resize(None, None, 0, 8, 8, 3, 16, 16, 0, ctypes.byref(rd), None) == 0
    assert lib.vrgdg_blend(None, None, None, 0, 0, 0.5, 0.5, None) == 0
    assert lib.vrgdg_lanczos4_resize_u8(None, None, 0, 8, 8, 16, 16, None, None, None, None, None, 0, None) == 0

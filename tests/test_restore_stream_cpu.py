"""The fused restore without a GPU: vrgdg_restore_blend's argument checks (each refusal happens before any CUDA call), the Python
wrapper's and restore_frames' refusals, and a guard that every k_restore instantiation has a case in tests/test_gpu_restore_stream.py."""
import ctypes

import pytest
import torch

import restore_matrix as rm


def _desc(nv, mode=2, roi=(0, 0, 8, 8), res=(16, 12), off=(0, 0)):
    return nv.ResizeDesc(mode, *roi, *res, *off)


def test_abi_rejects_bad_arguments_before_any_cuda_call(pkg):
    nv = pkg._native
    lib = nv.load_library()
    enh, orig, out = ctypes.c_void_p(256), ctypes.c_void_p(512), ctypes.c_void_p(1024)     # non-null, aligned, never dereferenced
    good = dict(enh=enh, orig=orig, out=out, B=2, n=2, He=8, We=8, Ce=3, H=12, W=16, Co=3, dtype=nv.F32, desc=_desc(nv))

    def call(**kw):
        a = dict(good, **kw)
        d = ctypes.byref(a["desc"]) if a["desc"] is not None else None
        return lib.vrgdg_restore_blend(a["enh"], a["orig"], a["out"], a["B"], a["n"], a["He"], a["We"], a["Ce"], a["H"], a["W"], a["Co"],
                                       a["dtype"], d, 0.3, 0.7, None)

    cases = [
        (dict(desc=None), b"null descriptor"),
        (dict(dtype=nv.U8BGR), b"float dtype"),
        (dict(dtype=7), b"float dtype"),
        (dict(H=-1), b"negative shape"),
        (dict(Co=2), b"channels"),
        (dict(Co=5), b"channels"),
        (dict(Ce=1), b"channels"),
        (dict(n=3), b"n_restored"),
        (dict(n=-1), b"n_restored"),
        (dict(desc=_desc(nv, mode=9)), b"unknown mode"),
        (dict(desc=_desc(nv, roi=(1, 0, 8, 8))), b"ROI"),
        (dict(desc=_desc(nv, roi=(0, 0, 8, 9))), b"ROI"),
        (dict(desc=_desc(nv, roi=(0, 0, 0, 8))), b"ROI"),
        (dict(desc=_desc(nv, res=(15, 12))), b"does not cover"),
        (dict(desc=_desc(nv, res=(16, 12), off=(1, 0))), b"does not cover"),
        (dict(desc=_desc(nv, res=(16, 12), off=(0, -1))), b"does not cover"),
        (dict(orig=None), b"null pointer"),
        (dict(out=None), b"null pointer"),
        (dict(enh=None), b"null pointer"),
        (dict(out=orig), b"in-place"),
        (dict(out=enh), b"in-place"),
        (dict(orig=ctypes.c_void_p(514)), b"aligned"),
    ]
    for kw, needle in cases:
        rc = call(**kw)
        msg = lib.vrgdg_last_error()
        want = nv.E_ALIGN if needle == b"aligned" else nv.E_INVALID
        assert rc == want and needle in msg and b"vrgdg_restore_blend" in msg, (kw, rc, msg)
        with pytest.raises(ValueError):
            nv.check(rc)
    # empty batches are a successful no-op before any CUDA call; no enhanced pointer is needed when no frame is blended
    assert call(enh=None, orig=None, out=None, B=0, n=0) == nv.VRGDG_OK
    assert call(B=0, n=0, Co=4, Ce=4, dtype=nv.BF16) == nv.VRGDG_OK


def test_wrapper_refuses_what_the_kernel_does_not_take(pkg):
    ops = pkg.ops
    x = torch.zeros(2, 4, 4, 3)
    with pytest.raises(RuntimeError, match="CUDA device"):           # host tensors never reach the library
        ops.restore_blend(x, x, "bicubic", 0.5, 0.5)


def test_restore_frames_keeps_its_errors_before_any_device_is_chosen(pkg):
    import importlib
    ve = importlib.import_module(pkg.__name__ + ".video_enhance")
    orig = torch.rand(3, 6, 8, 3)
    with pytest.raises(ValueError, match="non-empty"):
        ve.restore_frames(orig, orig[:0], 8, 6, "Stretch to dimensions", "Bilinear", 1.0)
    with pytest.raises(ValueError, match="source size 9x6"):
        ve.restore_frames(orig, orig, 9, 6, "Stretch to dimensions", "Bilinear", 1.0)


@pytest.mark.parametrize("fit", ["Stretch to dimensions", "Crop to fill", "Fit with letterbox (preserve all)"])
def test_restore_roi_is_the_one_restore_batch_resamples(pkg, oracle, fit):
    """the ROI handed to the fused kernel is the window oracle.restore_batch slices out of the working frame"""
    import importlib
    ve = importlib.import_module(pkg.__name__ + ".video_enhance")
    for (work_w, work_h), (sw, sh) in [((24, 24), (27, 21)), ((24, 24), (32, 21)), ((17, 13), (27, 21)), ((80, 80), (53, 37))]:
        x0, y0, w, h = ve._restore_roi(work_w, work_h, sw, sh, fit)
        x = torch.rand(1, work_h, work_w, 3, generator=torch.Generator().manual_seed(work_w))
        want = oracle.restore_batch(x, sw, sh, fit, "Nearest")
        got = oracle.resize_batch(x[:, y0:y0 + h, x0:x0 + w], sw, sh, "Stretch to dimensions", "Nearest")
        assert torch.equal(got, want), (fit, work_w, work_h, sw, sh)


def test_every_restore_kernel_has_a_gpu_case():
    inst = rm.instantiated()
    assert ("f32", "bicubic", 4, "vec") in inst and ("bf16", "area", 3, "scalar") in inst and not any(k[0] == "u8" for k in inst)
    assert len(inst) == len(rm.FLOAT_DTYPES) * len(rm.MODES) * 2 * 2
    reached = {rm.kernel_of(c) for c in rm.CASES}
    assert sorted(inst - reached) == [], "k_restore instantiations no GPU case runs"
    assert sorted(reached - inst) == [], "GPU cases name kernels launch_restore does not build"
    for key in inst:                          # each kernel with both enhanced channel counts and both geometries
        got = {(c.ce, c.geometry) for c in rm.CASES if rm.kernel_of(c) == key}
        assert got == {(ce, g) for ce in rm.CHANNELS for g in rm.GEOMETRIES}, key
    assert set(rm.N_RESTORED) >= {0, rm.FRAMES} and any(0 < n < rm.FRAMES for n in rm.N_RESTORED)
    assert set(rm.STRENGTHS) == {0.0, 0.35, 1.0}
    assert len({rm.case_id(c) for c in rm.CASES}) == len(rm.CASES)

"""CPU guard of the video-tools matrix (tests/test_gpu_video_tools_matrix.py): every k_adjust_point / k_adjust_box instantiation that
launch_adjust can select, every k_resize mode and channel count, and the blend, 4-channel LUT and codec kernels are reached by at
least one case for every frame dtype they are built for.  Also pins the area-resize window arithmetic to torch's CPU
F.interpolate(mode="area") at the sizes where an fp32 quotient picks the wrong window.  No GPU needed."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import video_tools_matrix as vtm


def test_instantiations_are_parsed():
    assert vtm.instantiated_dtypes("VRGDG_INSTANTIATE") == set(vtm.DTYPES)
    assert vtm.codec_dtypes() == set(vtm.FLOAT_DTYPES)
    inst = vtm.adjust_instantiations()
    # anchors: every window of the clarity pass in both positions, sharpen only with the 3 x 3 window and only last
    for dt in vtm.DTYPES:
        for k in (9, 7, 5, 3, 1):
            for last in (True, False):
                assert ("box", dt, k, 0, last, "scalar") in inst, (dt, k, last)
        assert ("box", dt, 3, 1, True, "vec") in inst and ("point", dt, True) in inst and ("point", dt, False) in inst
    assert not any(k[0] == "box" and k[3] == 1 and (k[2] != 3 or not k[4]) for k in inst)
    assert vtm.resize_modes() == set(vtm.RESIZE_MODES)
    assert ("f32", "area", 4) in vtm.resize_instantiations() and not any(k[0] == "u8" for k in vtm.resize_instantiations())
    assert vtm.blend_dtypes() == vtm.lut_rgba_dtypes() == set(vtm.FLOAT_DTYPES)


def test_adjust_matrix_reaches_every_instantiated_kernel():
    inst = vtm.adjust_instantiations()
    reached = set().union(*(vtm.adjust_kernels(c) for c in vtm.ADJUST_CASES))
    assert sorted(inst - reached, key=str) == [], "adjust kernel paths no matrix case runs"
    assert sorted(reached - inst, key=str) == [], "the selection mirror names kernels vrgdg_adjust.cuh does not build"


def test_adjust_shapes_select_every_window_in_both_aspects():
    for k in (1, 3, 5, 7, 9):
        shapes = [s for s in vtm.ADJUST_SHAPES.values() if vtm.blur_kernel(s[1], s[2]) == k]
        assert any(H < W for _, H, W in shapes) and any(W < H for _, H, W in shapes), k
        assert {W % 4 == 0 for _, H, W in shapes} == {True, False}, k
    # a multi-tile shape (16 x 64-pixel tiles) whose last tile is partial in both directions, on both store paths
    ragged = [(H, W) for _, H, W in vtm.ADJUST_SHAPES.values() if H > 2 * 16 and W > 2 * 64 and H % 16 and W % 64]
    assert {W % 4 == 0 for _, W in ragged} == {True, False}
    assert set(vtm.ADJUST_SETTINGS) >= {"pointwise", "clarity", "sharpen", "clarity_sharpen", "everything", "disabled"}


def test_resize_matrix_reaches_every_mode_dtype_and_channel_count():
    reached = {(c.dtype, c.mode, c.channels) for c in vtm.RESIZE_CASES}
    assert sorted(vtm.resize_instantiations() - reached) == []
    for key in vtm.resize_instantiations():
        geos = {c.geometry for c in vtm.RESIZE_CASES if (c.dtype, c.mode, c.channels) == key}
        assert set(vtm.RESIZE_GEOMETRIES) <= geos, key
    assert {c.dtype for c in vtm.BLEND_CASES} >= vtm.blend_dtypes()
    assert {c.dtype for c in vtm.LUT_RGBA_CASES} >= vtm.lut_rgba_dtypes()
    for dt in vtm.codec_dtypes():
        assert {c.direction for c in vtm.CODEC_CASES if c.dtype == dt} == set(vtm.CODEC_DIRECTIONS), dt
    ids = [vtm.resize_id(c) for c in vtm.RESIZE_CASES] + [vtm.adjust_id(c) for c in vtm.ADJUST_CASES]
    assert len(ids) == len(set(ids))


def test_error_bars():
    C = vtm.ResizeCase
    assert vtm.resize_bar(C("area", "bf16", 3, "stretch")) == 0 and vtm.resize_bar(C("nearest", "f16", 4, "crop")) == 0
    assert vtm.resize_bar(C("bicubic", "f32", 3, "roi")) == 2e-6
    assert vtm.resize_bar(C("bilinear", "f16", 3, "roi")) == 2.0 ** -11 and vtm.resize_bar(C("bilinear", "bf16", 3, "roi")) == 2.0 ** -8


def _fp32_bounds(o, n_in, n_out):
    """the window bounds as an fp32 quotient (what the area kernel computed before it used integers)"""
    f = np.float32
    return int(np.floor(f(o * n_in) / f(n_out))), int(np.ceil(f((o + 1) * n_in) / f(n_out)))


@pytest.mark.parametrize("n_in,n_out", vtm.AREA_STRIPS)
def test_area_window_bounds_match_torch_at_large_products(n_in, n_out):
    """integer bounds == torch's CPU area interpolation along either axis, where the fp32 quotient picks a different window"""
    x = torch.rand(n_in, generator=torch.Generator().manual_seed(n_in), dtype=torch.float64)
    want = torch.stack([x[a:b].mean() for a, b in (vtm.area_bounds(o, n_in, n_out) for o in range(n_out))])
    got_x = F.interpolate(x.view(1, 1, 1, n_in), size=(1, n_out), mode="area").view(-1)
    got_y = F.interpolate(x.view(1, 1, n_in, 1), size=(n_out, 1), mode="area").view(-1)
    assert torch.allclose(got_x, want, rtol=0, atol=1e-12) and torch.allclose(got_y, want, rtol=0, atol=1e-12)
    assert any(_fp32_bounds(o, n_in, n_out) != vtm.area_bounds(o, n_in, n_out) for o in range(n_out)), "no fp32 rounding here"
    for axis in ("x", "y"):
        for mode in ("area", "nearest"):
            for dt in vtm.FLOAT_DTYPES:
                assert vtm.ResizeCase(mode, dt, 3, "strip-%s-%d-%d" % (axis, n_in, n_out)) in vtm.RESIZE_CASES, (axis, mode, dt)


def test_fp32_window_of_4007_to_5009_reads_past_the_roi():
    """the case the strip's spare column / row guards: the last fp32 window ends one pixel past the source"""
    assert _fp32_bounds(5008, 4007, 5009) == (4006, 4008)
    assert vtm.area_bounds(5008, 4007, 5009) == (4006, 4007)

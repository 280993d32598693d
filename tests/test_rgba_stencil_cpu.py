"""RGBA frames through the three sharpener nodes, without a GPU: what the reference does with 4 channels (the oracle facts that
specify the feature), the argument checks of vrgdg_stencil3x3_ch, the nodes' refusal of the 4-channel torch paths, and a guard
that every launch_tile_rgba path has a case in tests/test_gpu_rgba_stencil.py."""
import ctypes

import pytest
import torch

import rgba_stencil_matrix as rsm


def _rgba(seed=0, shape=(2, 9, 11, 4)):
    return torch.rand(*shape, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("fn", ["unsharp_numpy", "unsharp_torch", "laplacian_numpy", "sobel_numpy"])
def test_reference_sharpens_every_channel_of_rgba_frames(oracle, fn):
    """the NumPy paths pad H and W only and the avg_pool2d unsharp pools per channel: each channel of the RGBA result is the RGB
    function's result on that channel"""
    f = getattr(oracle, fn)
    x = _rgba()
    y = f(x, 0.5)
    assert y.shape == x.shape
    assert torch.equal(y[..., :3], f(x[..., :3].contiguous(), 0.5))
    assert torch.equal(y[..., 3], f(x[..., 3:4].expand(-1, -1, -1, 3).contiguous(), 0.5)[..., 0])


@pytest.mark.parametrize("call", [lambda o, x: o.laplacian_torch(x, 0.5), lambda o, x: o.sobel_torch(x, 0.5),
                                  lambda o, x: o.film_grain(x, 0.04, 0.5), lambda o, x: o.adjust(x)],
                         ids=["laplacian_torch", "sobel_torch", "film_grain", "adjust"])
def test_reference_rejects_rgba_elsewhere(oracle, call):
    with pytest.raises(RuntimeError):
        call(oracle, _rgba())


def test_abi_rejects_unsupported_channel_layouts_without_a_gpu(pkg):
    nv = pkg._native
    lib = nv.load_library()
    src, dst = ctypes.c_void_p(256), ctypes.c_void_p(512)          # non-null, aligned, never dereferenced
    cases = [
        ((2, nv.F32, nv.STENCIL_BOX_UNSHARP), nv.E_INVALID, b"channels"),
        ((5, nv.F32, nv.STENCIL_BOX_UNSHARP), nv.E_INVALID, b"channels"),
        ((1, nv.F16, nv.STENCIL_SOBEL_CPU), nv.E_INVALID, b"channels"),
        ((4, nv.U8BGR, nv.STENCIL_BOX_UNSHARP), nv.E_UNSUPPORTED, b"uint8"),
        ((4, nv.F32, nv.STENCIL_LAPLACIAN_GPU), nv.E_UNSUPPORTED, b"takes 3 channels"),
        ((4, nv.BF16, nv.STENCIL_SOBEL_GPU), nv.E_UNSUPPORTED, b"takes 3 channels"),
        ((4, 7, nv.STENCIL_BOX_UNSHARP), nv.E_INVALID, b"dtype"),
        ((4, nv.F32, 9), nv.E_INVALID, b"bad op"),
    ]
    for (ch, dtype, op), code, needle in cases:
        rc = lib.vrgdg_stencil3x3_ch(src, dst, 1, 8, 8, ch, dtype, op, 0.5, nv.BORDER_REPLICATE, None)
        msg = lib.vrgdg_last_error()
        assert rc == code and needle in msg and b"vrgdg_stencil3x3_ch" in msg, (ch, dtype, op, rc, msg)
        with pytest.raises(ValueError):
            nv.check(rc)
    rc = lib.vrgdg_stencil3x3_ch(src, dst, 1, 8, 8, 4, nv.F32, nv.STENCIL_BOX_UNSHARP, 0.5, 2, None)
    assert rc == nv.E_INVALID and b"bad border" in lib.vrgdg_last_error()
    # empty batches are a successful no-op before any CUDA call, for both channel counts
    for ch in (3, 4):
        assert lib.vrgdg_stencil3x3_ch(None, None, 0, 8, 8, ch, nv.F32, nv.STENCIL_BOX_UNSHARP, 0.5, nv.BORDER_ZERO, None) == nv.VRGDG_OK


@pytest.mark.parametrize("key, method", [("FastLaplacianSharpen", "apply_laplacian"), ("FastSobelSharpen", "apply_sobel")])
def test_torch_path_nodes_refuse_rgba_before_choosing_a_device(pkg, key, method):
    node = pkg.NODE_CLASS_MAPPINGS[key]()
    with pytest.raises(ValueError, match="got 4 channels"):
        getattr(node, method)(_rgba(), 0.5, True)


@pytest.mark.parametrize("key", ["FastUnsharpSharpen", "FastLaplacianSharpen", "FastSobelSharpen"])
def test_sharpener_nodes_still_refuse_other_channel_counts(pkg, key):
    node = pkg.NODE_CLASS_MAPPINGS[key]()
    fn = getattr(node, node.FUNCTION)
    for c in (1, 2, 5):
        with pytest.raises(ValueError, match="3 or 4"):
            fn(_rgba(shape=(1, 6, 6, c)), 0.5, False)


def test_every_rgba_kernel_path_has_a_gpu_case():
    inst = rsm.instantiated()
    assert inst, "launch_tile_rgba selects no kernel"
    assert ("f32", rsm.BOX_UNSHARP, True) in inst and ("f16", rsm.SOBEL_CPU, False) in inst
    assert not any(op in (rsm.LAPLACIAN_GPU, rsm.SOBEL_GPU) for _, op, _ in inst)
    reached = {rsm.kernel_of(c) for c in rsm.CASES}
    assert sorted(inst - reached) == [], "launch_tile_rgba paths no GPU case runs"
    assert sorted(reached - inst) == [], "GPU cases name paths launch_tile_rgba does not build"
    # every path on the TMA loader and on the generic one
    for shape in rsm.SHAPES:
        assert {rsm.kernel_of(c) for c in rsm.CASES if c.shape == shape} == inst, shape
    assert {rsm.PATH[s] for s in rsm.SHAPES} == {"tma", "generic"}


def test_matrix_shapes_take_the_loaders_they_name():
    """the TMA map needs 16-byte aligned rows of at least 256 elements and 34 rows (vrgdg_abi.cu build_tmap)"""
    B, H, W = rsm.SHAPES["tma"]
    for es in (4, 2):
        assert (4 * W * es) % 16 == 0 and 4 * W >= 256 and H >= 34
    assert 4 * W > 2 * 240 and H > 2 * 32                          # several tiles in both directions
    B, H, W = rsm.SHAPES["small"]
    assert 4 * W < 256 and H < 34
    assert rsm.SHAPES["ragged"][2] % 2 == 1

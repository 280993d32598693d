"""RGBA frames through the fused post chain, without a GPU: what the reference's LUT -> sharpener composition does with 4 channels
(the oracle facts that specify the feature), the argument checks of vrgdg_chain_apply_ch, the refusals of VRGDG_B200_PostChain and
chain.PostChain before any device is chosen, and a guard that every launch_tile_rgba_lut path has a case in
tests/test_gpu_rgba_chain.py on both tile loaders."""
import ctypes
import os

import pytest
import torch

import rgba_chain_matrix as rcm
from helpers import natural_frames, write_big_cube


@pytest.fixture(scope="module")
def luts(oracle, tmp_path_factory):
    big = str(tmp_path_factory.mktemp("luts") / "big65.cube")
    write_big_cube(big, rcm.BIG_LUT_SIZE)
    return {name: oracle.parse_cube(path or big) for name, path in rcm.LUTS.items()}


def _rgba(B=2, H=9, W=11, seed=0):
    alpha = natural_frames(B, H, W, seed=seed + 1000)[..., 1:2]
    return torch.cat([natural_frames(B, H, W, seed=seed), alpha], dim=-1).contiguous()


@pytest.mark.parametrize("strength", rcm.LUT_STRENGTHS)
@pytest.mark.parametrize("lut", list(rcm.LUTS))
@pytest.mark.parametrize("pair", [None] + list(rcm.PAIRS), ids=lambda p: "lut_only" if p is None else "op%d-border%d" % p)
def test_reference_chain_on_rgba_is_rgb_chain_plus_filtered_alpha(oracle, luts, lut, strength, pair):
    """RGB of the RGBA composition = the RGB composition; alpha = the stencil on the LUT node's alpha, which is the input alpha at
    blend 1 and a*(1-blend) + a*blend otherwise"""
    x = _rgba(seed=3)
    L = dict(lut_data=luts[lut], strength=strength)
    st = None if pair is None else dict(op=pair[0], border=pair[1], strength=rcm.STRENGTH[pair[0]])
    y = oracle.chain_compose(x, lut=L, stencil=st)
    assert y.shape == x.shape
    assert torch.equal(y[..., :3], oracle.chain_compose(x[..., :3].contiguous(), lut=L, stencil=st))
    blend = strength / 10.0
    a = x[..., 3]
    lut_alpha = oracle.apply_lut(x, luts[lut], strength)[..., 3]
    assert torch.equal(lut_alpha, a if blend == 1.0 else a * (1.0 - blend) + a * blend)
    want = lut_alpha if st is None else oracle.CHAIN_STENCILS[pair](lut_alpha.unsqueeze(-1).expand(-1, -1, -1, 3).contiguous(),
                                                                     st["strength"])[..., 0]
    assert torch.equal(y[..., 3], want)


def _desc(nv, **kw):
    d = nv.ChainDesc()
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_abi_rejects_unsupported_rgba_chains_without_a_gpu(pkg):
    nv = pkg._native
    lib = nv.load_library()
    src, dst = ctypes.c_void_p(256), ctypes.c_void_p(512)          # non-null, aligned, never dereferenced
    unsharp = dict(stencil_op=nv.STENCIL_BOX_UNSHARP, stencil_strength=0.5)
    cases = [
        ((2, nv.F32, unsharp), nv.E_INVALID, b"channels"),
        ((5, nv.F16, unsharp), nv.E_INVALID, b"channels"),
        ((4, nv.U8BGR, unsharp), nv.E_UNSUPPORTED, b"uint8"),
        ((4, 7, unsharp), nv.E_INVALID, b"dtype"),
        ((4, nv.F32, dict(unsharp, grain_enabled=1)), nv.E_UNSUPPORTED, b"film grain"),
        ((4, nv.BF16, dict(colormatch_enabled=1)), nv.E_UNSUPPORTED, b"colour match"),
        ((4, nv.F16, dict(unsharp, post_grain_enabled=1)), nv.E_UNSUPPORTED, b"post grain"),
        ((4, nv.F32, dict(stencil_op=nv.STENCIL_LAPLACIAN_GPU)), nv.E_UNSUPPORTED, b"takes 3 channels"),
        ((4, nv.F16, dict(stencil_op=nv.STENCIL_SOBEL_GPU, stencil_border=nv.BORDER_ZERO)), nv.E_UNSUPPORTED, b"takes 3 channels"),
        ((4, nv.F32, dict(stencil_op=9)), nv.E_INVALID, b"bad stencil op"),
        ((4, nv.F32, dict(unsharp, stencil_border=2)), nv.E_INVALID, b"bad border"),
        ((4, nv.F32, dict(unsharp, lut_enabled=1)), nv.E_INVALID, b"LUT"),
    ]
    for (ch, dtype, fields), code, needle in cases:
        rc = lib.vrgdg_chain_apply_ch(src, dst, 1, 8, 8, ch, dtype, ctypes.byref(_desc(nv, **fields)), None)
        msg = lib.vrgdg_last_error()
        assert rc == code and needle in msg, (ch, dtype, fields, rc, msg)
        with pytest.raises(ValueError):
            nv.check(rc)
    # the stencil reads neighbours: no in-place run
    rc = lib.vrgdg_chain_apply_ch(src, src, 1, 8, 8, 4, nv.F32, ctypes.byref(_desc(nv, **unsharp)), None)
    assert rc == nv.E_INVALID and b"in place" in lib.vrgdg_last_error()
    rc = lib.vrgdg_chain_apply_ch(src, dst, 1, 8, 8, 4, nv.F32, None, None)
    assert rc == nv.E_INVALID and b"null descriptor" in lib.vrgdg_last_error()
    # empty batches are a successful no-op before any CUDA call, for both channel counts
    for ch in (3, 4):
        assert lib.vrgdg_chain_apply_ch(None, None, 0, 8, 8, ch, nv.F32, ctypes.byref(_desc(nv, **unsharp)), None) == nv.VRGDG_OK


def _node_call(pkg, images, **kw):
    args = dict(grain_intensity=0.0, saturation_mix=0.5, match_strength=1.0, lut_name="none", lut_strength=10.0, sharpen="unsharp",
                sharpen_strength=0.5, use_gpu=False, batch_size=8)
    args.update(kw)
    return pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_PostChain"]().apply_chain(images, **args)


@pytest.mark.parametrize("kw, needle", [
    (dict(grain_intensity=0.04), "grain_intensity"),
    (dict(reference_image=torch.rand(1, 9, 11, 3)), "reference_image"),
    (dict(sharpen="laplacian", use_gpu=True), "use_gpu=True"),
    (dict(sharpen="sobel", use_gpu=True), "use_gpu=True"),
], ids=["grain", "colour_match", "laplacian_torch_path", "sobel_torch_path"])
def test_post_chain_node_refuses_rgba_stages_before_choosing_a_device(pkg, kw, needle):
    with pytest.raises(ValueError, match=needle):
        _node_call(pkg, _rgba(), **kw)


def test_post_chain_node_still_refuses_other_channel_counts(pkg):
    for c in (1, 2, 5):
        with pytest.raises(ValueError, match="3 or 4"):
            _node_call(pkg, torch.rand(1, 6, 6, c))


def test_post_chain_node_inputs_are_unchanged(pkg):
    req = pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_PostChain"].INPUT_TYPES()
    assert list(req["required"]) == ["images", "grain_intensity", "saturation_mix", "match_strength", "lut_name", "lut_strength", "sharpen",
                                     "sharpen_strength", "use_gpu", "batch_size"]
    assert list(req["optional"]) == ["reference_image"]


@pytest.mark.parametrize("stages, needle", [
    (dict(grain=dict(intensity=0.04, saturation_mix=0.5)), "grain"),
    (dict(post_grain=dict(intensity=0.03, saturation_mix=0.7), stencil=dict(op=1, strength=0.5)), "post_grain"),
    (dict(stencil=dict(op=3, strength=0.3, border=1)), "torch conv2d"),
    (dict(stencil=dict(op=5, strength=0.3, border=1)), "torch conv2d"),
], ids=["grain", "post_grain", "laplacian_torch_path", "sobel_torch_path"])
def test_post_chain_refuses_rgba_stages_before_any_upload(pkg, stages, needle):
    chain = pkg.chain.PostChain(device="cuda:0", **stages)       # no LUT / reference: nothing touches the device here
    x = _rgba()
    with pytest.raises(ValueError, match=needle):
        chain(x)
    with pytest.raises(ValueError, match=needle):
        chain.run_host(x)
    with pytest.raises(ValueError, match=needle):
        chain.make_fn()(torch.device("cuda", 0))(x, 0)


def test_every_rgba_chain_kernel_path_has_a_gpu_case():
    inst = rcm.instantiated()
    assert inst, "launch_tile_rgba_lut selects no kernel"
    assert ("f32", 1, True) in inst and ("bf16", 4, False) in inst
    assert not any(op in (3, 5) for _, op, _ in inst)
    reached = {rcm.kernel_of(c) for c in rcm.CASES} - {None}
    assert sorted(inst - reached) == [], "launch_tile_rgba_lut paths no GPU case runs"
    assert sorted(reached - inst) == [], "GPU cases name paths launch_tile_rgba_lut does not build"
    # every path on the TMA loader and on the generic one, with every LUT and both blend regimes
    for shape in rcm.SHAPES:
        assert {rcm.kernel_of(c) for c in rcm.CASES if c.shape == shape} - {None} == inst, shape
    assert {rcm.PATH[s] for s in rcm.SHAPES} == {"tma", "generic"}
    for lut in rcm.LUTS:
        for s in rcm.LUT_STRENGTHS:
            assert {rcm.kernel_of(c) for c in rcm.CASES if c.lut == lut and c.strength == s} - {None} == inst, (lut, s)
    assert {c.stages for c in rcm.CASES} == set(rcm.STAGES)
    assert all(os.path.exists(p) for p in rcm.LUTS.values() if p)

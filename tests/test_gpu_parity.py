"""GPU parity tests: CUDA kernels (through the C ABI / node classes) vs golden vectors produced by the reference's
own source (tests/golden/make_golden.py) and vs the CPU oracle.  Tolerances: bit-exact for the 3D LUT, the
ext-noise grain arithmetic and the u8 codecs; 1e-5 max-abs (fp32) for sharpen / colour match / fused chains
(BASELINE.json north_star)."""
import json
import hashlib
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN, LUTS, load_golden, natural_frames, t, white_frames

pytestmark = pytest.mark.gpu
TOL = 1e-5


def maxdiff(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max())


@pytest.fixture(scope="module")
def meta():
    with open(os.path.join(GOLDEN, "reference_meta.json"), encoding="utf-8") as fh:
        return json.load(fh)


def test_library_loads_on_sm90(pkg, cuda_device):
    lib = pkg._native.load_library()
    import ctypes
    sm, major, minor = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    pkg._native.check(lib.vrgdg_device_info(ctypes.byref(sm), ctypes.byref(major), ctypes.byref(minor)))
    assert (major.value, minor.value) == (9, 0) and sm.value >= 100


# ------------------------------------------------------------------------------------------------------
# 3D LUT — bit-exact
# ------------------------------------------------------------------------------------------------------
def test_lut_node_bit_exact_all_fixtures(pkg, cuda_device):
    g = load_golden("lut")
    node = pkg.VRGDG_LUTS()
    x, xn = t(g["x"]), t(g["xn"])
    n = 0
    for fname in sorted(os.listdir(LUTS)):
        if not fname.endswith(".cube"):
            continue
        key = fname.split(".")[0].replace(" ", "_")
        before = pkg._native.launch_count()
        o10 = node.apply_lut(x, fname, "auto", 10.0)[0]
        assert pkg._native.launch_count() > before, "no kernel launched"
        assert o10.device.type == "cpu" and o10.dtype == torch.float32
        assert torch.equal(o10, t(g[f"{key}__s10"])), fname
        assert torch.equal(node.apply_lut(x, fname, "cuda", 3.5)[0], t(g[f"{key}__s3p5"])), fname
        assert torch.equal(node.apply_lut(xn, fname, "cpu", 10.0)[0], t(g[f"{key}__nat"])), fname
        n += 1
    assert n >= 4


def test_lut_strength_zero_returns_input(pkg, cuda_device):
    x = white_frames(1, 8, 8)
    out = pkg.VRGDG_LUTS().apply_lut(x, "B200 Vintage 33.cube", "auto", 0.0)[0]
    assert torch.equal(out, x)


def test_lut_rgba_fp16_domain(pkg, cuda_device):
    g = load_golden("lut")
    node = pkg.VRGDG_LUTS()
    v33 = "B200 Vintage 33.cube"
    assert torch.equal(node.apply_lut(t(g["x4"]), v33, "auto", 10.0)[0], t(g["v33_rgba"]))
    assert torch.equal(node.apply_lut(t(g["x4"]), v33, "auto", 3.5)[0], t(g["v33_rgba_s3p5"]))
    # fp16 frames: reference rounds LUT output to fp16 (and blends in fp16); we round once -> <= 1 fp16 ulp
    o16 = node.apply_lut(t(g["x"]).half(), v33, "auto", 10.0)[0]
    assert o16.dtype == torch.float16
    assert torch.equal(o16, t(g["v33_fp16"]))                       # single rounding of identical fp32 values
    o16b = node.apply_lut(t(g["x"]).half(), v33, "auto", 3.5)[0]
    assert maxdiff(o16b, t(g["v33_fp16_s3p5"])) <= 2 * 2.0 ** -11
    # non-unit DOMAIN_MIN/MAX
    dom = pkg.VRGDG_LUTS._parse_cube_file(os.path.join(GOLDEN, "domain_5.cube"))
    xd = t(g["x"]).to(cuda_device)
    out = pkg.VRGDG_LUTS._apply_cube_lut(xd, dom["lut"], dom["domain_min"], dom["domain_max"])
    assert torch.equal(out.cpu(), t(g["domain5_s10"]))


def test_lut_identity_full_size_property(pkg, cuda_device):
    """size-independent property at 4K: an identity table reproduces the input (to fp32 rounding of the lerp)."""
    S = 33
    ax = torch.linspace(0, 1, S)
    b, gg, r = torch.meshgrid(ax, ax, ax, indexing="ij")
    ident = torch.stack([r, gg, b], dim=-1).contiguous().to(cuda_device)
    x = natural_frames(2, 2160, 3840, seed=9, device=cuda_device)
    out = pkg.ops.lut3d_apply(x, ident, [0, 0, 0], [1, 1, 1], 1.0, 0.0)
    assert maxdiff(out, x) < 5e-7


# ------------------------------------------------------------------------------------------------------
# grain
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["a", "odd"])
def test_grain_ext_noise_bit_exact(pkg, cuda_device, tag):
    g = load_golden("grain")
    x, z = t(g[f"x_{tag}"]).to(cuda_device), t(g[f"z_{tag}"]).to(cuda_device)
    o = pkg.ops.grain(x, 0.5, 0.5, 1.0 - 0.5, seed=0, ext_noise=z)
    assert torch.equal(o.cpu(), t(g[f"out_{tag}_i50_s50"]))
    o = pkg.ops.grain(x, 0.04, 0.37, 1.0 - 0.37, seed=0, ext_noise=z)
    assert torch.equal(o.cpu(), t(g[f"out_{tag}_i04_s37"]))


def test_config1_512x512_intensity_half(pkg, cuda_device, meta, oracle):
    """BASELINE.json configs[0]: FastFilmGrain on 1x512x512, intensity 0.5, same N(0,1) tensor as the reference drew."""
    x = torch.rand(1, 512, 512, 3, generator=torch.Generator().manual_seed(0))
    torch.manual_seed(123)
    z = torch.randn_like(x)
    sha = lambda a: hashlib.sha256(a.contiguous().numpy().tobytes()).hexdigest()
    out = pkg.ops.grain(x.to(cuda_device), 0.5, 0.5, 0.5, seed=0, ext_noise=z.to(cuda_device)).cpu()
    if sha(x) == meta["config1"]["x_sha256"] and sha(z) == meta["config1"]["z_sha256"]:
        assert sha(out) == meta["config1"]["out_sha256"]
        assert torch.equal(out[0, 100:132, 200:232], t(load_golden("config1_crop")["out_crop"]))
    else:  # a different torch CPU RNG on this box: fall back to the oracle on the tensors drawn here
        assert torch.equal(out, oracle.film_grain(x, 0.5, 0.5, 0, noise=z))


def test_grain_noise_distribution(pkg, cuda_device):
    z = pkg.ops.grain_noise(2, 512, 512, seed=1234, device=cuda_device).double()
    n = z.numel()
    assert abs(float(z.mean())) < 4.0 / n ** 0.5
    assert abs(float(z.var()) - 1.0) < 0.01
    assert abs(float((z ** 4).mean()) - 3.0) < 0.05          # kurtosis of N(0,1)
    assert abs(float((z ** 3).mean())) < 0.02
    assert float(z.abs().max()) > 4.5                        # tails exist
    # channels of a pixel and neighbouring pixels are uncorrelated
    zr, zg, zb = z[..., 0].flatten(), z[..., 1].flatten(), z[..., 2].flatten()
    for a, b in ((zr, zg), (zr, zb), (zg, zb), (zr[:-1], zr[1:]), (zg[:-1], zb[1:])):
        assert abs(float((a * b).mean())) < 5.0 / a.numel() ** 0.5
    # frames differ, seeds differ
    assert float((z[0] - z[1]).abs().mean()) > 0.5
    z2 = pkg.ops.grain_noise(1, 512, 512, seed=1235, device=cuda_device).double()
    assert float((z[0] - z2[0]).abs().mean()) > 0.5
    # empirical CDF vs N(0,1) at a few quantiles
    flat = z.flatten()
    for q, p in ((-1.0, 0.158655), (0.0, 0.5), (1.0, 0.841345), (2.0, 0.977250)):
        assert abs(float((flat < q).double().mean()) - p) < 2e-3


def test_grain_partition_invariance(pkg, cuda_device):
    """the reference's own invariant (tests/test_standalone_video_enhancer.py:39-60): batch boundaries do not matter."""
    nv = pkg._native
    frames = torch.full((4, 12, 16, 3), 0.5, device=cuda_device)
    for mode in (nv.SEED_PER_FRAME, nv.SEED_PER_CLIP):
        whole = pkg.ops.grain(frames, 0.04, 0.5, 0.5, seed=42, frame0=100, seed_mode=mode)
        split = torch.cat([pkg.ops.grain(frames[:2], 0.04, 0.5, 0.5, seed=42, frame0=100, seed_mode=mode),
                           pkg.ops.grain(frames[2:], 0.04, 0.5, 0.5, seed=42, frame0=102, seed_mode=mode)])
        assert torch.equal(whole, split)
        assert not torch.equal(whole[0], whole[1])
    # vector path (hw % 4 == 0) and scalar path (odd hw) draw the same noise for the same pixel index
    a = pkg.ops.grain_noise(1, 6, 8, seed=5, device=cuda_device)            # reference stream
    xa = torch.full((1, 6, 8, 3), 0.5, device=cuda_device)
    ga = pkg.ops.grain(xa, 0.1, 1.0, 0.0, seed=5)
    assert torch.allclose(ga, (0.5 + 0.1 * a * torch.tensor([2.0, 1.0, 3.0], device=cuda_device)).clamp(0, 1), atol=1e-6)


def test_film_grain_node_reproducible_and_batch_size_free(pkg, cuda_device):
    x = white_frames(5, 33, 47, seed=3)
    node = pkg.FastFilmGrain()
    torch.manual_seed(77)
    a = node.apply_grain(x, 0.04, 0.5, 4)[0]
    torch.manual_seed(77)
    b = node.apply_grain(x, 0.04, 0.5, 0)[0]
    torch.manual_seed(78)
    c = node.apply_grain(x, 0.04, 0.5, 2)[0]
    assert a.shape == x.shape and a.device.type == "cpu"
    assert torch.equal(a, b) and not torch.equal(a, c)
    d = (a - x)
    assert 0.02 < float(d[..., 1].std()) < 0.06          # ~ intensity * N(0,1) on green (clamping shrinks it slightly)
    assert float(a.min()) >= 0.0 and float(a.max()) <= 1.0


def test_seeded_grain_arithmetic_matches_reference_on_its_noise(pkg, cuda_device):
    g = load_golden("effects")
    out = pkg.ops.grain(t(g["frames"]).to(cuda_device), 0.04, 0.5, 0.5, seed=0, ext_noise=t(g["z"]).to(cuda_device))
    assert torch.equal(out.cpu(), t(g["whole"]))
    out = pkg.ops.grain(t(g["sharp_only"]).to(cuda_device), 0.04, 0.5, 0.5, seed=0, ext_noise=t(g["ze"]).to(cuda_device))
    assert torch.equal(out.cpu(), t(g["eff"]))


# ------------------------------------------------------------------------------------------------------
# 3x3 stencils
# ------------------------------------------------------------------------------------------------------
STENCIL_CASES = [("unsharp", "FastUnsharpSharpen", "apply_unsharp"), ("laplacian", "FastLaplacianSharpen", "apply_laplacian"),
                 ("sobel", "FastSobelSharpen", "apply_sobel")]


@pytest.mark.parametrize("key,cls,fn", STENCIL_CASES)
def test_stencil_nodes_vs_reference(pkg, cuda_device, key, cls, fn):
    g = load_golden("stencil")
    node = getattr(pkg, cls)()
    x = t(g["x"])
    o = getattr(node, fn)(x, 0.5, False)[0]
    assert pkg._native.last_tile_path() == "tma"          # 72 x 96 frames take the TMA path
    assert o.device.type == "cpu"
    # fp32 frames, NumPy-path semantics: the kernels evaluate in the reference's order with one rounding per op -> bit-exact
    assert torch.equal(o, t(g[f"{key}_np"]))
    assert maxdiff(getattr(node, fn)(x, 0.5, True)[0], t(g[f"{key}_torch"])) <= TOL      # torch conv/pool paths: tolerance
    assert torch.equal(getattr(node, fn)(t(g["x_odd"]), 1.3, False)[0], t(g[f"{key}_np_odd"]))
    assert pkg._native.last_tile_path() == "generic"      # 37 x 53: rows not 16-byte aligned
    assert torch.equal(getattr(node, fn)(t(g["x_tiny"]), 0.7, False)[0], t(g[f"{key}_np_tiny"]))
    assert torch.equal(getattr(node, fn)(t(g["x_one"]), 0.7, False)[0], t(g[f"{key}_np_one"]))


def test_unsharp_strength_10_and_half_precision(pkg, cuda_device):
    g = load_golden("stencil")
    x = t(g["x"])
    assert torch.equal(pkg.FastUnsharpSharpen().apply_unsharp(x, 10.0, False)[0], t(g["unsharp_np_s10"]))
    assert torch.equal(pkg.FastUnsharpSharpen().apply_unsharp(x, 0.5, True)[0], t(g["unsharp_torch"]))     # avg_pool2d sums in the same order
    for dt, ulp in ((torch.float16, 2.0 ** -11), (torch.bfloat16, 2.0 ** -8)):
        xh = x.to(dt)
        oh = pkg.FastUnsharpSharpen().apply_unsharp(xh, 0.5, False)[0]
        assert oh.dtype == dt
        ref = pkg.FastUnsharpSharpen().apply_unsharp(xh.float(), 0.5, False)[0]
        assert maxdiff(oh, ref) <= ulp        # fp32 arithmetic on the rounded input, one final rounding


@pytest.mark.parametrize("H,W,B,dtype", [(1080, 1920, 3, torch.float32), (2160, 3840, 1, torch.float32), (1080, 1920, 2, torch.float16),
                                         (1000, 1004, 2, torch.float32), (34, 88, 2, torch.float32)])
def test_stencil_tma_equals_generic_loader_full_size(pkg, cuda_device, H, W, B, dtype):
    """size-independent property: the TMA-staged path and the bounds-checked loader produce identical frames."""
    nv = pkg._native
    x = natural_frames(B, H, W, seed=H + W, dtype=dtype, device=cuda_device)
    for op, border in ((nv.STENCIL_BOX_UNSHARP, nv.BORDER_REPLICATE), (nv.STENCIL_SOBEL_GPU, nv.BORDER_ZERO), (nv.STENCIL_LAPLACIAN_CPU, nv.BORDER_REPLICATE)):
        a = pkg.ops.stencil3x3(x, op, 0.7, border)
        assert nv.last_tile_path() == "tma"
        os.environ["VRGDG_NO_TMA"] = "1"
        try:
            b = pkg.ops.stencil3x3(x, op, 0.7, border)
            assert nv.last_tile_path() == "generic"
        finally:
            del os.environ["VRGDG_NO_TMA"]
        assert torch.equal(a, b)
    # constant frames are fixed points of every sharpener with replicate borders (except sobel-gpu's +1e-6)
    c = torch.full((1, H, W, 3), 0.25, dtype=dtype, device=cuda_device)
    for op in (nv.STENCIL_BOX_UNSHARP, nv.STENCIL_LAPLACIAN_CPU, nv.STENCIL_LAPLACIAN_GPU, nv.STENCIL_SOBEL_CPU):
        assert maxdiff(pkg.ops.stencil3x3(c, op, 1.5, nv.BORDER_REPLICATE), c) <= 1e-6


def test_unsharp_full_size_vs_oracle_crop(pkg, cuda_device, oracle):
    """4K frame through the TMA path; the oracle checks three crops incl. image corners (finishes in < 1 s)."""
    x = natural_frames(1, 2160, 3840, seed=77)
    o = pkg.ops.stencil3x3(x.to(cuda_device), pkg._native.STENCIL_BOX_UNSHARP, 0.5, pkg._native.BORDER_REPLICATE).cpu()
    ref = oracle.unsharp_numpy(x, 0.5)
    assert torch.equal(o, ref)


# ------------------------------------------------------------------------------------------------------
# colour match
# ------------------------------------------------------------------------------------------------------
def test_lab_moments_vs_oracle(pkg, cuda_device, oracle):
    g = load_golden("colormatch")
    x = t(g["x"])
    sums = pkg.ops.lab_moments(x.to(cuda_device)).cpu()
    ref = oracle.lab_moments_f64(x)
    n = float(ref[0, 0])
    assert torch.equal(sums[:, 0], ref[:, 0])
    assert float((sums[:, 1:4] - ref[:, 1:4]).abs().max()) / n < 5e-5          # mean Lab within 5e-5 units (scale 0..100)
    assert torch.allclose(sums[:, 4:7], ref[:, 4:7], rtol=5e-6, atol=0.0)
    # row sharding adds up
    a = pkg.ops.lab_moments(x.to(cuda_device), 0, 30).cpu()
    b = pkg.ops.lab_moments(x.to(cuda_device), 30, 42).cpu()
    assert torch.allclose(a + b, sums, rtol=1e-12, atol=1e-9)
    # deterministic
    assert torch.equal(pkg.ops.lab_moments(x.to(cuda_device)).cpu(), sums)


def test_colormatch_node_vs_reference(pkg, cuda_device):
    g = load_golden("colormatch")
    node = pkg.ColorMatchToReference()
    o = node.match_color(t(g["x"]), t(g["ref"]), 1.0, 1)[0]
    assert o.shape == g["x"].shape and o.device.type == "cpu"
    assert maxdiff(o, t(g["out_t100"])) <= TOL
    assert maxdiff(node.match_color(t(g["x"]), t(g["ref"]), 0.6, 2)[0], t(g["out_t60"])) <= TOL
    # CUDA in -> stays on the device outside ComfyUI
    oc = node.match_color(t(g["x"]).to(cuda_device), t(g["ref"]), 1.0, 1)[0]
    assert oc.device.type == "cuda" and maxdiff(oc, t(g["out_t100"])) <= TOL


# ------------------------------------------------------------------------------------------------------
# fused chains
# ------------------------------------------------------------------------------------------------------
def _lut33(pkg):
    return pkg.VRGDG_LUTS._parse_cube_file(os.path.join(LUTS, "B200 Vintage 33.cube"))


def test_chain_grain_lut_unsharp_vs_reference_composition(pkg, cuda_device):
    """BASELINE.json configs[1] arithmetic: FastFilmGrain(ext z) -> VRGDG_LUTS(33^3) -> FastUnsharpSharpen, one kernel."""
    nv = pkg._native
    g = load_golden("chain")
    chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=0), lut=dict(lut_data=_lut33(pkg), strength=10.0),
                                stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5, border=nv.BORDER_REPLICATE), device=cuda_device)
    before = nv.launch_count()
    out = chain(t(g["x"]).to(cuda_device), ext_noise=t(g["z"]).to(cuda_device))
    assert nv.launch_count() - before == 1 and nv.last_tile_path() == "tma"
    assert torch.equal(out.cpu(), t(g["grain_lut_unsharp"]))      # every stage reproduces the reference's roundings: bit-exact chain
    # the arithmetic variant the benchmark runs (FMA-contracted blend / lerps), fed the same noise: same bar
    fast = chain(t(g["x"]).to(cuda_device), ext_noise=t(g["z"]).to(cuda_device), fast_math=True)
    assert maxdiff(fast, t(g["grain_lut_unsharp"])) <= TOL and maxdiff(fast, out) <= 2e-6
    chain2 = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=0), lut=dict(lut_data=_lut33(pkg), strength=6.0),
                                 stencil=dict(op=nv.STENCIL_SOBEL_CPU, strength=0.3), device=cuda_device)
    assert torch.equal(chain2(t(g["x"]).to(cuda_device), ext_noise=t(g["z"]).to(cuda_device)).cpu(), t(g["grain_lut60_sobel"]))


def test_full_chain_with_colormatch_vs_reference_composition(pkg, cuda_device):
    """configs[3] arithmetic: grain -> colour match -> LUT -> unsharp."""
    nv = pkg._native
    g = load_golden("chain")
    x, z = t(g["x"]).to(cuda_device), t(g["z"]).to(cuda_device)
    # the moments pass must see the same grained frames -> feed them explicitly for this ext-noise comparison
    grained = pkg.ops.grain(x, 0.04, 0.5, 0.5, seed=0, ext_noise=z)
    ref_sums = pkg.ops.lab_moments(t(g["ref"]).to(cuda_device))
    params = pkg.ops.colormatch_params(pkg.ops.lab_moments(grained), ref_sums)
    d = nv.ChainDesc()
    d.grain_enabled, d.grain_intensity, d.grain_sat, d.grain_one_minus_sat = 1, 0.04, 0.5, 0.5
    d.colormatch_enabled, d.cm_params, d.cm_t, d.cm_one_minus_t = 1, params.data_ptr(), 1.0, 0.0
    lut = _lut33(pkg)
    lut_dev = pkg.ops.pack_lut(lut["lut"], cuda_device)
    import ctypes
    d.lut_enabled, d.lut, d.lut_size = 1, lut_dev.data.data_ptr(), 33
    d.lut_dmin, d.lut_dspan = (ctypes.c_float * 3)(0, 0, 0), (ctypes.c_float * 3)(1, 1, 1)
    d.lut_blend, d.lut_one_minus_blend = 1.0, 0.0
    d.stencil_op, d.stencil_strength, d.stencil_border = nv.STENCIL_BOX_UNSHARP, 0.5, nv.BORDER_REPLICATE
    out = pkg.ops.chain_apply(x, d, ext_noise=z)
    assert maxdiff(out, t(g["grain_cm_lut_unsharp"])) <= TOL


def test_chain_philox_equals_separate_kernels(pkg, cuda_device):
    """The fused kernel and the three standalone kernels draw the same noise and agree to fp32 rounding."""
    nv = pkg._native
    x = natural_frames(3, 136, 248, seed=5, device=cuda_device)
    lut = _lut33(pkg)
    chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), lut=dict(lut_data=lut, strength=10.0),
                                stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=cuda_device)
    fused = chain(x, first_frame=10)
    a = pkg.ops.grain(x, 0.04, 0.5, 0.5, seed=42, frame0=10)
    b = pkg.ops.lut3d_apply(a, lut["lut"].to(cuda_device), [0, 0, 0], [1, 1, 1], 1.0, 0.0)
    c = pkg.ops.stencil3x3(b, nv.STENCIL_BOX_UNSHARP, 0.5, nv.BORDER_REPLICATE)
    assert maxdiff(fused, c) <= 2e-6
    # shard invariance: frames 1..2 processed alone with first_frame=11 equal the tail of the full batch
    assert torch.equal(chain(x[1:].contiguous(), first_frame=11), fused[1:])
    # pointwise-only chain (no stencil) goes through k_point
    pw = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), lut=dict(lut_data=lut, strength=10.0), device=cuda_device)
    assert maxdiff(pw(x, first_frame=10), b) <= 1e-6
    # generic loader agrees with TMA for the fused kernel too
    os.environ["VRGDG_NO_TMA"] = "1"
    try:
        assert torch.equal(chain(x, first_frame=10), fused)
    finally:
        del os.environ["VRGDG_NO_TMA"]


def test_effects_batch_unsharp_then_seeded_grain(pkg, cuda_device):
    """_apply_effects_batch (EnhancerNodes.py:278-294): unsharp -> per-frame seeded grain, fused via post_grain."""
    nv = pkg._native
    g = load_golden("effects")
    xe = t(g["xe"]).to(cuda_device)
    sharp = pkg.ops.stencil3x3(xe, nv.STENCIL_BOX_UNSHARP, 0.8, nv.BORDER_REPLICATE)
    assert torch.equal(sharp.cpu(), t(g["sharp_only"]))
    chain = pkg.chain.PostChain(stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.8),
                                post_grain=dict(intensity=0.04, saturation_mix=0.5, seed=42, seed_mode=nv.SEED_PER_FRAME), device=cuda_device)
    fused = chain(xe, first_frame=7)
    two_step = pkg.ops.grain(sharp, 0.04, 0.5, 0.5, seed=42, frame0=7, seed_mode=nv.SEED_PER_FRAME)
    assert maxdiff(fused, two_step) <= 1e-6
    # partition invariance of the fused effect chain
    parts = torch.cat([chain(xe[:1].contiguous(), first_frame=7), chain(xe[1:].contiguous(), first_frame=8)])
    assert torch.equal(parts, fused)


def test_config2_shape_fp16_chain_consistency(pkg, cuda_device):
    """configs[1] at (reduced batch) full frame size: 8 x 1080p fp16 fused == separate kernels within fp16 rounding."""
    nv = pkg._native
    x = natural_frames(8, 1080, 1920, seed=2, dtype=torch.float16, device=cuda_device)
    lut = _lut33(pkg)
    chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), lut=dict(lut_data=lut, strength=10.0),
                                stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=cuda_device)
    fused = chain(x)
    assert nv.last_tile_path() == "tma"
    xf = x.float()
    a = pkg.ops.grain(xf, 0.04, 0.5, 0.5, seed=42)
    b = pkg.ops.lut3d_apply(a, lut["lut"].to(cuda_device), [0, 0, 0], [1, 1, 1], 1.0, 0.0)
    c = pkg.ops.stencil3x3(b, nv.STENCIL_BOX_UNSHARP, 0.5, nv.BORDER_REPLICATE)
    assert maxdiff(fused, c) <= 2.0 ** -11 + 1e-6
    assert float(fused.float().min()) >= 0 and float(fused.float().max()) <= 1


# ------------------------------------------------------------------------------------------------------
# wire format, host streaming, errors
# ------------------------------------------------------------------------------------------------------
def test_u8_bgr_codecs_bit_exact(pkg, cuda_device):
    g = load_golden("u8")
    f = pkg.ops.u8bgr_to_rgb(t(g["bgr"]).to(cuda_device))
    assert torch.equal(f.cpu(), t(g["rgb_float"]))
    u = pkg.ops.rgb_to_u8bgr(t(g["float_in"]).to(cuda_device))
    assert torch.equal(u.cpu(), t(g["bgr_out"]))


def test_host_streaming_matches_device_call(pkg, cuda_device):
    nv = pkg._native
    x = natural_frames(7, 64, 96, seed=8)
    chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=1), stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5),
                                device=cuda_device)
    whole = chain(x.to(cuda_device)).cpu()
    streamed = chain.run_host(x.pin_memory(), chunk_frames=3)
    assert streamed.device.type == "cpu" and torch.equal(streamed, whole)


def test_error_mapping(pkg, cuda_device):
    with pytest.raises(RuntimeError):
        pkg.ops.grain(white_frames(1, 4, 4), 0.1, 0.5, 0.5, seed=1)               # CPU tensor: no CPU path
    with pytest.raises(ValueError):
        pkg.ops.stencil3x3(torch.zeros(1, 4, 4, 2, device=cuda_device), 1, 0.5)   # not RGB
    with pytest.raises(ValueError):
        pkg.ops.stencil3x3(torch.zeros(1, 4, 4, 3, device=cuda_device), 9, 0.5)   # bad op -> VRGDG_E_INVALID
    with pytest.raises(ValueError):
        pkg.VRGDG_LUTS().apply_lut(white_frames(1, 4, 4), "No LUT files found", "auto", 10.0)
    with pytest.raises(FileNotFoundError):
        pkg.VRGDG_LUTS().apply_lut(white_frames(1, 4, 4), "missing.cube", "auto", 10.0)
    with pytest.raises(ValueError):
        pkg.VRGDG_LUTS().apply_lut(torch.zeros(4, 4, 3), "B200 Vintage 33.cube", "auto", 10.0)
    # empty batch is a no-op
    e = pkg.ops.grain(torch.zeros(0, 4, 4, 3, device=cuda_device), 0.1, 0.5, 0.5, seed=1)
    assert e.shape == (0, 4, 4, 3)


# ------------------------------------------------------------------------------------------------------
# full-size, size-independent properties for the colour-match configs (configs[2], configs[3])
# ------------------------------------------------------------------------------------------------------
def test_colormatch_full_size_self_reference_is_identity(pkg, cuda_device):
    """4K frames matched to THEMSELVES (each frame its own reference, batch-wise reference) must come back unchanged:
    (lab-mu)/sd*sd+mu == lab up to rounding, then Lab->RGB inverts RGB->Lab.  Exercises moments + params + apply at 4K."""
    x = natural_frames(2, 2160, 3840, seed=31, device=cuda_device)
    x[1] = (x[1] * 0.6 + 0.2)
    out = pkg.ColorMatchToReference().match_color(x, x, 1.0, 2)[0]
    assert out.device.type == "cuda" and maxdiff(out, x) <= 2e-5     # Lab round trip in fp32 (oracle: 2e-5 on the same test)
    half = pkg.ColorMatchToReference().match_color(x, x[:1].contiguous(), 0.0, 1)[0]   # strength 0: pure Lab round trip
    assert maxdiff(half, x) <= 2e-5


def test_colormatch_moves_statistics_onto_the_reference(pkg, cuda_device, oracle):
    """after a full-strength match the frame's LAB mean/std equal the reference's (what the node is for), at 1080p"""
    x = natural_frames(2, 1080, 1920, seed=32, device=cuda_device)
    ref = (natural_frames(1, 720, 1280, seed=33, device=cuda_device) * torch.tensor([0.9, 0.7, 0.8], device=cuda_device) + 0.05).clamp(0, 1)
    out = pkg.ColorMatchToReference().match_color(x, ref, 1.0, 1)[0]
    def stats(t):
        s = pkg.ops.lab_moments(t).cpu()
        n, m = s[:, :1], s[:, 1:4] / s[:, :1]
        return m, ((s[:, 4:7] - s[:, 1:4] * m) / (n - 1)).sqrt()
    mo, so = stats(out)
    mr, sr = stats(ref)
    inside = float(((out > 0) & (out < 1)).float().mean())
    assert inside > 0.98                                  # little clipping, otherwise the statistics cannot match
    assert float((mo - mr).abs().max()) < 0.5 and float((so / sr - 1).abs().max()) < 0.03


def test_full_chain_with_colormatch_partition_invariance(pkg, cuda_device):
    """configs[3] shape property: grain -> colour match -> LUT -> unsharp on shards == on the whole clip (frame-sharded dp)."""
    nv = pkg._native
    x = natural_frames(4, 270, 480, seed=34, device=cuda_device)
    ref = natural_frames(1, 135, 240, seed=35, device=cuda_device)
    lut = _lut33(pkg)
    mk = lambda: pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), colormatch=dict(reference_image=ref, strength=1.0),
                                     lut=dict(lut_data=lut, strength=10.0), stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=cuda_device)
    whole = mk()(x, first_frame=0)
    parts = torch.cat([mk()(x[:1].contiguous(), first_frame=0), mk()(x[1:].contiguous(), first_frame=1)])
    assert torch.equal(whole, parts)
    # and equals the unfused sequence of kernels
    a = pkg.ops.grain(x, 0.04, 0.5, 0.5, seed=42)
    params = pkg.ops.colormatch_params(pkg.ops.lab_moments(a), pkg.ops.lab_moments(ref))
    b = pkg.ops.colormatch_apply(a, params, 1.0, 0.0)
    c = pkg.ops.lut3d_apply(b, lut["lut"], [0, 0, 0], [1, 1, 1], 1.0, 0.0)
    d = pkg.ops.stencil3x3(c, nv.STENCIL_BOX_UNSHARP, 0.5, nv.BORDER_REPLICATE)
    assert maxdiff(whole, d) <= 5e-6


# ------------------------------------------------------------------------------------------------------
# uint8 BGR wire format fused into the kernels (SURVEY 8f rank 1): bytes in, bytes out, 6 B/px of traffic
# ------------------------------------------------------------------------------------------------------
def test_u8_frames_through_every_stage_bit_exact(pkg, cuda_device):
    """reference: _frames_to_tensor -> node(s) -> _tensor_to_frames on cv2 BGR bytes; ours: one kernel on the bytes.
    Truncating clip(x*255) makes bytes sensitive to the last bit, so this only holds because every stage reproduces the
    reference's roundings."""
    nv = pkg._native
    g = load_golden("u8chain")
    x = t(g["bgr_in"]).to(cuda_device)
    z = t(g["z"]).to(cuda_device)
    lut = _lut33(pkg)
    assert x.dtype == torch.uint8
    out = pkg.ops.grain(x, 0.04, 0.5, 0.5, seed=0, ext_noise=z)
    assert out.dtype == torch.uint8 and torch.equal(out.cpu(), t(g["grain_only"]))
    assert torch.equal(pkg.ops.lut3d_apply(x, lut["lut"], [0, 0, 0], [1, 1, 1], 1.0, 0.0).cpu(), t(g["lut_only"]))
    u = pkg.ops.stencil3x3(x, nv.STENCIL_BOX_UNSHARP, 0.5, nv.BORDER_REPLICATE)
    assert nv.last_tile_path() == "tma" and torch.equal(u.cpu(), t(g["unsharp_only"]))
    os.environ["VRGDG_NO_TMA"] = "1"
    try:
        assert torch.equal(pkg.ops.stencil3x3(x, nv.STENCIL_BOX_UNSHARP, 0.5, nv.BORDER_REPLICATE), u)
    finally:
        del os.environ["VRGDG_NO_TMA"]
    chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=0), lut=dict(lut_data=lut, strength=10.0),
                                stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=cuda_device)
    fused = chain(x, ext_noise=z)
    assert fused.dtype == torch.uint8 and torch.equal(fused.cpu(), t(g["grain_lut_unsharp"]))
    # the production arithmetic (contracted FMAs) may flip a byte only where x*255 sits within ~1e-5 of an integer
    fast = chain(x, ext_noise=z, fast_math=True).cpu().int()
    d = (fast - t(g["grain_lut_unsharp"]).int()).abs()
    assert int(d.max()) <= 1 and float((d > 0).float().mean()) < 1e-3


def test_u8_chain_equals_float_chain_on_decoded_frames(pkg, cuda_device):
    """bytes path == explicit codec kernels around the fp32 path (same generator, same arithmetic), at 1080p"""
    nv = pkg._native
    x = (natural_frames(3, 1080, 1920, seed=72, device=cuda_device) * 255).round().clamp(0, 255).to(torch.uint8)
    lut = _lut33(pkg)
    chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=5), lut=dict(lut_data=lut, strength=10.0),
                                stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=cuda_device)
    a = chain(x, first_frame=4)
    assert nv.last_tile_path() == "tma"
    b = pkg.ops.rgb_to_u8bgr(chain(pkg.ops.u8bgr_to_rgb(x), first_frame=4))
    d = (a.int() - b.int()).abs()
    assert int(d.max()) <= 1 and float((d > 0).float().mean()) < 1e-4      # identical kernels; only FMA contraction order could differ
    # post-grain on bytes (enhancer chain) and partition invariance
    eff = pkg.chain.PostChain(stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.8),
                              post_grain=dict(intensity=0.04, saturation_mix=0.5, seed=42, seed_mode=nv.SEED_PER_FRAME), device=cuda_device)
    whole = eff(x, first_frame=7)
    parts = torch.cat([eff(x[:2].contiguous(), first_frame=7), eff(x[2:].contiguous(), first_frame=9)])
    assert torch.equal(whole, parts)
    ref = pkg.ops.rgb_to_u8bgr(eff(pkg.ops.u8bgr_to_rgb(x), first_frame=7))
    d2 = (whole.int() - ref.int()).abs()
    assert int(d2.max()) <= 1 and float((d2 > 0).float().mean()) < 1e-4


# ------------------------------------------------------------------------------------------------------
# function-level drop-ins (video_tools.py: the reference's module-level helper names)
# ------------------------------------------------------------------------------------------------------
def test_video_tools_helpers_match_reference_outputs(pkg, cuda_device):
    import importlib
    vt = importlib.import_module("comfyui-vrgamedevgirl_b200.video_tools")
    g = load_golden("lut")
    out = vt._apply_lut_tensor(t(g["x"]), "B200 Vintage 33.cube", 7.0, "cpu")          # VRGDG_LUTVideoTools.py:172-185
    assert out.device.type == "cpu" and torch.equal(out, t(g["tensor_fn_s7"]))
    e = load_golden("effects")
    st = {"sharpen_enabled": True, "sharpen_strength": 0.8, "grain_enabled": False, "use_gpu": False}
    assert torch.equal(vt._apply_effects_batch(t(e["xe"]), st, 7), t(e["sharp_only"]))   # EnhancerNodes.py:278-294, numpy-path unsharp
    st2 = dict(st, grain_enabled=True, grain_intensity=0.04, saturation_mix=0.5, seed=42)
    whole = vt._apply_effects_batch(t(e["xe"]), st2, 7)
    parts = torch.cat([vt._apply_effects_batch(t(e["xe"])[:1], st2, 7), vt._apply_effects_batch(t(e["xe"])[1:], st2, 8)])
    assert whole.device.type == "cpu" and torch.equal(whole, parts)                      # the reference's own batch-boundary invariant
    d = (whole - t(e["sharp_only"]))
    assert 0.02 < float(d[..., 1].std()) < 0.06 and not torch.equal(whole, t(e["sharp_only"]))
    assert torch.equal(vt._apply_unsharp(t(e["xe"]), 0.8, False), t(e["sharp_only"]))
    assert vt._apply_unsharp(t(e["xe"]), 0.0, False) is not None and torch.equal(vt._apply_seeded_grain(t(e["xe"]), 0.0, 0.5, 1, 0), t(e["xe"]))
    u = load_golden("u8")
    assert torch.equal(vt._frames_to_tensor(list(u["bgr"])).cpu(), t(u["rgb_float"]))     # LUTVideoTools.py:736-743
    frames = vt._tensor_to_frames(t(u["float_in"]))
    assert np.array_equal(np.stack(frames), u["bgr_out"])                                 # :746-752, truncation
    fg = vt._apply_film_grain_tensor(t(e["xe"]), 0.04, 0.5, "cpu", seed=11)
    assert torch.equal(fg, vt._apply_film_grain_tensor(t(e["xe"]), 0.04, 0.5, "cpu", seed=11)) and not torch.equal(fg, t(e["xe"]))


# ------------------------------------------------------------------------------------------------------
# "adjust" pass (SURVEY 8f rank 2): _apply_adjust_tensor, VRGDG_LUTVideoTools.py:307-391
# ------------------------------------------------------------------------------------------------------
def test_adjust_tensor_bit_exact_all_cases(pkg, cuda_device, meta, oracle):
    import importlib
    vt = importlib.import_module("comfyui-vrgamedevgirl_b200.video_tools")
    g = load_golden("adjust")
    x = t(g["x"])
    for name, st in meta["adjust_cases"].items():
        before = pkg._native.launch_count()
        out = vt._apply_adjust_tensor(x, st, "cpu")
        assert pkg._native.launch_count() > before
        assert out.device.type == "cpu"
        if float(st.get("vignette", 0)) > 0:
            # the vignette mask goes through torch.sqrt, which on CPU is MKL VML's < 1 ulp (not correctly rounded) routine:
            # 0.7 % of the mask values differ from IEEE sqrt by 1 ulp -> tolerance instead of equality for this one stage
            assert maxdiff(out, t(g[name])) <= 2e-7 and float((out != t(g[name])).float().mean()) < 0.02, name
        else:
            assert torch.equal(out, t(g[name])), name
    # frames narrower than the 9x9 window: the blur kernel shrinks (5x7 -> 5)
    tiny = vt._apply_adjust_tensor(x[:, :5, :7].contiguous(), meta["adjust_cases"]["everything"], "cpu")
    assert maxdiff(tiny, t(g["tiny_5x7"])) <= 2e-7
    novig = dict(meta["adjust_cases"]["everything"], vignette=0)
    assert torch.equal(vt._apply_adjust_tensor(x, novig, "cpu"), oracle.adjust(x, novig))     # every other stage together: bit-exact
    # device-resident call keeps the result on the GPU; non-numeric / out-of-range sliders are normalised like the reference
    dev_out = vt._apply_adjust_tensor(x.to(cuda_device), {"exposure": "abc", "contrast": 1e9, "sharpen": -5}, cuda_device)
    ref = vt._apply_adjust_tensor(x, {"contrast": 100.0}, "cpu")
    assert dev_out.device.type == "cuda" and torch.equal(dev_out.cpu(), ref)


def test_adjust_full_size_properties(pkg, cuda_device, oracle):
    """1080p: neutral settings == clamp; and the oracle agrees on a whole frame with every stage on (1 frame: ~1 s of CPU)."""
    import importlib
    vt = importlib.import_module("comfyui-vrgamedevgirl_b200.video_tools")
    x = natural_frames(1, 1080, 1920, seed=91) * 1.2 - 0.1
    assert torch.equal(vt._apply_adjust_tensor(x, {}, "cpu"), oracle.adjust(x, {}))       # neutral sliders still round through (x-0.5)*1+0.5
    assert torch.equal(vt._apply_adjust_tensor(x, {"enabled": False, "exposure": 50}, "cpu"), x.clamp(0, 1))
    st = {"temperature": 20, "exposure": 10, "contrast": 15, "saturation": 10, "highlights": -20, "shadows": 20, "sharpen": 40, "clarity": 50,
          "fade": 10}
    assert torch.equal(vt._apply_adjust_tensor(x, st, "cpu"), oracle.adjust(x, st))
    stv = dict(st, vignette=30)
    assert maxdiff(vt._apply_adjust_tensor(x, stv, "cpu"), oracle.adjust(x, stv)) <= 2e-7
    # uint8 frames: decode -> adjust -> encode in the kernels == codecs around the float path
    u8 = (x.clamp(0, 1) * 255).round().to(torch.uint8).to(cuda_device)
    a = pkg.ops.adjust(u8, vt._adjust_desc(st, 1080, 1920))
    b = pkg.ops.rgb_to_u8bgr(pkg.ops.adjust(pkg.ops.u8bgr_to_rgb(u8), vt._adjust_desc(st, 1080, 1920)))
    assert a.dtype == torch.uint8 and torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------
# resize / restore around the enhancer (SURVEY 8f rank 3): VRGDG_VideoEnhanceNodes.py:54-106, :404-418
# ------------------------------------------------------------------------------------------------------
RESIZE_TOL = 2e-6      # bilinear / bicubic: fp32 rounding (ATen's own CPU kernels differ by this much between thread counts)


def test_resize_batch_all_modes_vs_reference(pkg, cuda_device, meta):
    import importlib
    ve = importlib.import_module("comfyui-vrgamedevgirl_b200.video_enhance")
    g = load_golden("resize")
    x = t(g["x"])
    for key, method, fit, tw, th in meta["resize_cases"]:
        before = pkg._native.launch_count()
        out = ve._resize_batch(x, tw, th, fit, method)
        assert pkg._native.launch_count() == before + 1, key          # interpolate + crop / pad + clamp: one launch
        ref = t(g[key])
        assert out.shape == ref.shape and out.device.type == "cpu", key
        if method in ("Nearest", "Area"):
            assert torch.equal(out, ref), key
        else:
            assert maxdiff(out, ref) <= RESIZE_TOL, (key, maxdiff(out, ref))
    up = t(g["Bicubic|Fit|80x80"])
    assert maxdiff(ve._restore_batch(up, 96, 54, "Fit with letterbox (preserve all)", "Bicubic (recommended)"), t(g["restore_letterbox"])) <= RESIZE_TOL
    assert maxdiff(ve._restore_batch(up, 96, 54, "Stretch to dimensions", "Bilinear"), t(g["restore_stretch"])) <= RESIZE_TOL
    # RGBA input: alpha is dropped like images[..., :3]; unknown method names fall back to bicubic (:45-51)
    rgba = torch.cat([x, torch.ones_like(x[..., :1])], dim=-1)
    assert torch.equal(ve._resize_batch(rgba, 160, 72, "Stretch to dimensions", "Nearest"), t(g["Nearest|Stretch|160x72"]))
    assert torch.equal(ve._resize_batch(x, 160, 72, "Stretch to dimensions", "???"), ve._resize_batch(x, 160, 72, "Stretch to dimensions", "Bicubic (recommended)"))
    with pytest.raises(ValueError):
        ve._resize_batch(x[0], 10, 10, "Stretch to dimensions", "Nearest")
    # half precision frames: same geometry, fp16 rounding of the result
    h = ve._resize_batch(x.to(cuda_device).half(), 160, 72, "Stretch to dimensions", "Bilinear")
    assert h.dtype == torch.float16 and h.device.type == "cuda"
    assert maxdiff(h.float().cpu(), t(g["Bilinear|Stretch|160x72"])) <= 1.5e-3


def test_resize_full_size_vs_oracle_and_properties(pkg, cuda_device, oracle):
    """720p -> 1080p and back (the enhancer's prepare / restore shapes), against the oracle on whole frames (~1 s CPU), plus
    size-independent properties: identity at equal size, letterbox bars are exact zeros, restore(crop ROI) == resize of the crop."""
    import importlib
    ve = importlib.import_module("comfyui-vrgamedevgirl_b200.video_enhance")
    x = natural_frames(2, 720, 1280, seed=93) * 1.1 - 0.05
    for method in ("Nearest", "Bilinear", "Bicubic (recommended)", "Area"):
        up = ve._resize_batch(x, 1920, 1088, "Crop to fill", method)
        ref = oracle.resize_batch(x, 1920, 1088, "Crop to fill", method)
        assert up.shape == ref.shape == (2, 1088, 1920, 3)
        assert (torch.equal(up, ref) if method in ("Nearest", "Area") else maxdiff(up, ref) <= RESIZE_TOL), method
        down = ve._restore_batch(up, 1280, 720, "Crop to fill", method)
        refd = oracle.restore_batch(ref, 1280, 720, "Crop to fill", method)
        assert (torch.equal(down, refd) if method == "Nearest" else maxdiff(down, refd) <= 2 * RESIZE_TOL), method
        same = ve._resize_batch(x, 1280, 720, "Stretch to dimensions", method)
        assert maxdiff(same, x.clamp(0, 1)) <= (0 if method in ("Nearest", "Area") else 1e-6), method
    lb = ve._resize_batch(x, 1024, 1024, "Fit with letterbox (preserve all)", "Bicubic (recommended)")
    assert lb.shape == (2, 1024, 1024, 3)
    assert float(lb[:, :224].abs().max()) == 0.0 and float(lb[:, 800:].abs().max()) == 0.0       # 1024x576 content, 224-row bars
    assert maxdiff(lb, oracle.resize_batch(x, 1024, 1024, "Fit with letterbox (preserve all)", "Bicubic (recommended)")) <= RESIZE_TOL
    back = ve._restore_batch(lb, 1280, 720, "Fit with letterbox (preserve all)", "Bicubic (recommended)")
    assert maxdiff(back, ve._resize_batch(lb[:, 224:800].contiguous(), 1280, 720, "Stretch to dimensions", "Bicubic (recommended)")) == 0.0


def test_restore_frames_blend_bit_exact(pkg, cuda_device, oracle):
    import importlib
    ve = importlib.import_module("comfyui-vrgamedevgirl_b200.video_enhance")
    orig = natural_frames(5, 54, 96, seed=95) * 1.2 - 0.1
    enh = natural_frames(3, 54, 96, seed=96)                                   # sampler returned 2 frames fewer, same size
    out = ve.restore_frames(orig, enh, 96, 54, "Stretch to dimensions", "Nearest", 0.65)
    ref = orig.clone()
    ref[:3] = orig[:3] * (1.0 - 0.65) + oracle.restore_batch(enh, 96, 54, "Stretch to dimensions", "Nearest") * 0.65
    assert torch.equal(out, ref.clamp(0, 1))                                   # :410-418, tail frames keep the (clamped) original
    assert torch.equal(out[3:], orig[3:].clamp(0, 1))
    a, b = orig[:3].to(cuda_device), enh.to(cuda_device)
    assert torch.equal(pkg.ops.blend(a, b, 1.0, 0.0), a.clamp(0, 1)) and torch.equal(pkg.ops.blend(a, b, 0.0, 1.0), b)
    with pytest.raises(ValueError):
        pkg.ops.blend(a, b[:2], 0.5, 0.5)


# ------------------------------------------------------------------------------------------------------
# the enhancer's cv2 Lanczos4 resize of uint8 frames (SURVEY 8f rank 3): EnhancerNodes.py:213-230
# ------------------------------------------------------------------------------------------------------
def test_resize_frames_lanczos4_bit_exact_vs_cv2(pkg, cuda_device, meta):
    import importlib
    vt = importlib.import_module("comfyui-vrgamedevgirl_b200.video_tools")
    g = load_golden("lanczos")
    for name, ow, oh in meta["lanczos_cases"]:
        src = g[name + "_in"]
        before = pkg._native.launch_count()
        out = vt._resize_frames([src, src], ow, oh)
        assert len(out) == 2 and out[0].dtype == np.uint8 and out[0].shape == g[name].shape, name
        assert np.array_equal(out[0], g[name]) and np.array_equal(out[1], g[name]), name
        if name == "same":
            assert out[0] is src and pkg._native.launch_count() == before           # pass-through, like the reference (:221-222)
        else:
            assert pkg._native.launch_count() == before + 2, name                    # horizontal + vertical pass for the whole group
    # mixed sizes in one call: each group of equal-sized frames is one batch
    a, b = g["noise_up_in"], g["noise_odd_in"]
    mixed = vt._resize_frames([a, b, a], 106, 74)
    assert np.array_equal(mixed[0], g["noise_up"]) and np.array_equal(mixed[2], g["noise_up"]) and mixed[1].shape == (74, 106, 3)
    with pytest.raises(ValueError):
        vt._resize_frames([a.astype(np.float32)], 10, 10)
    with pytest.raises(ValueError):
        pkg.ops.resize_lanczos4_u8(torch.zeros(1, 4, 4, 3, dtype=torch.uint8), 8, 8)     # CPU tensor: no CPU path


def test_lanczos4_full_size_vs_oracle_and_properties(pkg, cuda_device, oracle):
    """720p -> 1080p (the enhancer's upscale) against the oracle on a whole frame (~1 s CPU); plus size-independent properties at
    4K: a constant frame stays constant (weights sum to 2048 only approximately -> within 1 code), frames are independent of the
    batch they travel in, small scratch budgets (frame groups) give identical bytes."""
    rng = np.random.default_rng(12)
    f = torch.from_numpy(rng.integers(0, 256, (2, 720, 1280, 3), dtype=np.uint8)).to(cuda_device)
    out = pkg.ops.resize_lanczos4_u8(f, 1080, 1920)
    assert out.shape == (2, 1080, 1920, 3)
    assert np.array_equal(out[1].cpu().numpy(), oracle.resize_lanczos4_u8(f[1].cpu().numpy(), 1920, 1080))
    down = pkg.ops.resize_lanczos4_u8(out, 405, 721)                                       # odd sizes: scalar vertical pass (721*3 % 4 != 0)
    assert np.array_equal(down[0].cpu().numpy(), oracle.resize_lanczos4_u8(out[0].cpu().numpy(), 721, 405))
    big = torch.full((3, 1080, 1920, 3), 200, dtype=torch.uint8, device=cuda_device)
    big[1] = torch.from_numpy(rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8)).to(cuda_device)
    up = pkg.ops.resize_lanczos4_u8(big, 2160, 3840)
    assert int((up[0].int() - 200).abs().max()) <= 1 and torch.equal(up[0], up[2])
    assert torch.equal(up[1], pkg.ops.resize_lanczos4_u8(big[1:2], 2160, 3840)[0])
    assert torch.equal(up, pkg.ops.resize_lanczos4_u8(big, 2160, 3840, max_scratch_bytes=1))   # one frame per launch pair
    assert pkg.ops.resize_lanczos4_u8(big[:0], 50, 60).shape == (0, 50, 60, 3)


# ------------------------------------------------------------------------------------------------------
# ragged shapes: every loader / border / tail path against the oracle (small frames: the oracle needs milliseconds)
# ------------------------------------------------------------------------------------------------------
def test_random_ragged_shapes_bit_exact_vs_oracle(pkg, cuda_device, oracle):
    """40 random shapes (1 x 1 up to 3 x 75 x 530: below / above the 34-row and 256-element TMA limits, widths that are not a
    multiple of 4, single rows and columns): the exact-arithmetic kernels must equal the oracle bit for bit on all of them, the
    TMA and the bounds-checked loaders must agree, and the uint8 path must equal codecs around the float path."""
    nv = pkg._native
    rng = np.random.default_rng(2024)
    lut = _lut33(pkg)
    olut = oracle.parse_cube(os.path.join(LUTS, "B200 Vintage 33.cube"))
    shapes = [(1, 1, 1), (1, 1, 7), (2, 9, 1), (1, 2, 2), (1, 34, 86), (1, 35, 88), (1, 33, 340), (2, 70, 84), (1, 36, 529)]
    while len(shapes) < 40:
        shapes.append((int(rng.integers(1, 4)), int(rng.integers(1, 76)), int(rng.integers(1, 531))))
    seen_tma = False
    for i, (B, H, W) in enumerate(shapes):
        x = torch.from_numpy(rng.random((B, H, W, 3), dtype=np.float32) * 1.2 - 0.1)
        z = torch.from_numpy(rng.standard_normal((B, H, W, 3)).astype(np.float32))
        xd, zd = x.to(cuda_device), z.to(cuda_device)
        tag = (B, H, W)
        # stencils, NumPy-path semantics (edge-replicated border)
        for op, fn in ((nv.STENCIL_BOX_UNSHARP, oracle.unsharp_numpy), (nv.STENCIL_LAPLACIAN_CPU, oracle.laplacian_numpy),
                       (nv.STENCIL_SOBEL_CPU, oracle.sobel_numpy))[i % 3:i % 3 + 1]:
            got = pkg.ops.stencil3x3(xd, op, 0.7, nv.BORDER_REPLICATE)
            seen_tma |= nv.last_tile_path() == "tma"
            assert torch.equal(got.cpu(), fn(x, 0.7)), (tag, op)
            os.environ["VRGDG_NO_TMA"] = "1"
            try:
                assert torch.equal(pkg.ops.stencil3x3(xd, op, 0.7, nv.BORDER_REPLICATE), got), (tag, op, "generic loader")
            finally:
                del os.environ["VRGDG_NO_TMA"]
        # LUT node arithmetic, strength blend
        lut_dev = pkg.ops.pack_lut(lut["lut"], cuda_device)
        got = pkg.ops.lut3d_apply(xd, lut_dev, [0, 0, 0], [1, 1, 1], 0.35, 1.0 - 0.35)
        assert torch.equal(got.cpu(), oracle.apply_lut(x, olut, 3.5)), tag
        # fused chain on the reference's noise
        chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=0), lut=dict(lut_data=lut, strength=10.0),
                                    stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5, border=nv.BORDER_REPLICATE), device=cuda_device)
        got = chain(xd, ext_noise=zd)
        assert torch.equal(got.cpu(), oracle.chain_grain_lut_unsharp(x, z, 0.04, 0.5, olut, 10.0, 0.5)), tag
        # uint8 BGR frames through the same chain == decode -> float chain -> encode
        u8 = torch.from_numpy(rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)).to(cuda_device)
        a = chain(u8, ext_noise=zd)
        b = pkg.ops.rgb_to_u8bgr(chain(pkg.ops.u8bgr_to_rgb(u8), ext_noise=zd))
        assert a.dtype == torch.uint8 and torch.equal(a, b), tag
    assert seen_tma                                                             # the list covers both loaders


def test_batches_beyond_2G_elements_use_64bit_indexing(pkg, cuda_device):
    """Maximum sizes (configs[2] / [3] are 6.4 G elements per call): 88 x 4K fp16 frames = 2.19 G elements > 2^31.  Every kernel
    family must treat the LAST frames exactly as it treats them alone (absolute frame index passed for the grain)."""
    nv = pkg._native
    B, H, W = 88, 2160, 3840
    assert B * H * W * 3 > 2 ** 31
    x = torch.empty((B, H, W, 3), dtype=torch.float16, device=cuda_device)
    gen = torch.Generator(device=cuda_device).manual_seed(7)
    for b0 in range(0, B, 8):
        x[b0:b0 + 8] = torch.rand((min(8, B - b0), H, W, 3), generator=gen, device=cuda_device, dtype=torch.float32).half()
    tail = x[B - 2:].clone()
    lut = _lut33(pkg)
    chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), lut=dict(lut_data=lut, strength=10.0),
                                stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=cuda_device)
    full = chain(x)                                                     # k_tile, TMA coordinates with a large frame index
    assert nv.last_tile_path() == "tma"
    assert torch.equal(full[B - 2:], chain(tail, first_frame=B - 2))
    del full
    g = pkg.ops.grain(x, 0.04, 0.5, 0.5, seed=9)                        # k_point
    assert torch.equal(g[B - 2:], pkg.ops.grain(tail, 0.04, 0.5, 0.5, seed=9, frame0=B - 2))
    del g
    u = pkg.ops.stencil3x3(x, nv.STENCIL_SOBEL_GPU, 0.3, nv.BORDER_ZERO)
    assert torch.equal(u[B - 2:], pkg.ops.stencil3x3(tail, nv.STENCIL_SOBEL_GPU, 0.3, nv.BORDER_ZERO))
    del u
    sums = pkg.ops.lab_moments(x)                                       # per-frame reductions
    assert torch.equal(sums[B - 2:], pkg.ops.lab_moments(tail))
    params = pkg.ops.colormatch_params(sums, sums[:1].contiguous())
    cm = pkg.ops.colormatch_apply(x, params, 1.0, 0.0)
    assert torch.equal(cm[B - 2:], pkg.ops.colormatch_apply(tail, params[B - 2:].contiguous(), 1.0, 0.0))


def test_enhance_frames_bytes_in_bytes_out(pkg, cuda_device, oracle):
    """The enhancer's per-batch data path (EnhancerNodes.py:415-420) fused on the device == the four helpers called one after the
    other (bytes), and == the oracle for the deterministic part (Lanczos4 -> /255 -> unsharp -> truncating encode)."""
    import importlib
    vt = importlib.import_module("comfyui-vrgamedevgirl_b200.video_tools")
    rng = np.random.default_rng(21)
    frames = [rng.integers(0, 256, (90, 160, 3), dtype=np.uint8) for _ in range(5)]
    st = {"sharpen_enabled": True, "sharpen_strength": 0.6, "grain_enabled": True, "grain_intensity": 0.05, "saturation_mix": 0.4, "seed": 77,
          "use_gpu": False}
    before = pkg._native.launch_count()
    fused = vt.enhance_frames(frames, 240, 136, st, frame_start=12)
    assert pkg._native.launch_count() == before + 3                                 # Lanczos h + v, unsharp + grain on the bytes
    steps = vt._tensor_to_frames(vt._apply_effects_batch(vt._frames_to_tensor(vt._resize_frames(frames, 240, 136)), st, 12))
    assert len(fused) == 5 and all(np.array_equal(a, b) for a, b in zip(fused, steps))
    nograin = dict(st, grain_enabled=False)
    got = vt.enhance_frames(frames, 240, 136, nograin, 0)
    ref = oracle.tensor_to_frames(oracle.effects_batch(oracle.frames_to_tensor(oracle.resize_frames(frames, 240, 136)), nograin, 0))
    assert all(np.array_equal(a, b) for a, b in zip(got, ref))
    same = vt.enhance_frames(frames, 160, 90, dict(nograin, use_gpu=True), 0)       # no resize, torch-path border
    ref2 = oracle.tensor_to_frames(oracle.unsharp_torch(oracle.frames_to_tensor(frames), 0.6))     # avg_pool2d path (:240-250)
    assert all(np.array_equal(a, b) for a, b in zip(same, ref2))
    assert vt.enhance_frames([], 10, 10, st) == []
    mixed = vt.enhance_frames([frames[0], frames[1][:45]], 80, 46, nograin, 0)      # mixed sizes: helper-by-helper route
    assert mixed[0].shape == mixed[1].shape == (46, 80, 3)

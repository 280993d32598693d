"""RGBA IMAGE batches through the fused post chain (vrgdg_chain_apply_ch: k_lut_rgba, k_tile<T, 0, ., 4> and the one-pass
k_tile<T, ST_LUT, true, 4>) against the oracle composition, channel by channel against the 3-channel fused chain, against the
two-kernel composition, and through the VRGDG_B200_PostChain node: host and CUDA batches against VRGDG_LUTS -> Fast*Sharpen, and
sharded over two workers.  The cases come from tests/rgba_chain_matrix.py, whose CPU guard checks that they reach every
launch_tile_rgba_lut path on both tile loaders."""
import functools
import importlib
import os

import pytest
import torch

import rgba_chain_matrix as rcm
from helpers import natural_frames, write_big_cube

pytestmark = pytest.mark.gpu

TORCH = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
NODE_LUT = "B200 Vintage 33.cube"


@pytest.fixture(scope="module")
def env(pkg, oracle, tmp_path_factory):
    big = str(tmp_path_factory.mktemp("luts") / "big65.cube")
    write_big_cube(big, rcm.BIG_LUT_SIZE)
    paths = {name: path or big for name, path in rcm.LUTS.items()}
    return dict(lut={n: pkg.VRGDG_LUTS._parse_cube_file(p) for n, p in paths.items()},
                olut={n: oracle.parse_cube(p) for n, p in paths.items()}, chains={})


@functools.lru_cache(maxsize=None)
def _rgba(dtype, shape, seed=0):
    """natural RGB frames and a spatially coherent alpha plane of its own (an edge-free alpha would hide a wrong neighbour)"""
    B, H, W = rcm.SHAPES[shape] if isinstance(shape, str) else shape
    alpha = natural_frames(B, H, W, seed=seed + B * 7 + H * 3 + W + 1000)[..., 1:2]
    x = torch.cat([natural_frames(B, H, W, seed=seed + B * 7 + H * 3 + W), alpha], dim=-1).contiguous()
    return x.to(TORCH[dtype])


def _chain(pkg, env, dev, lut, strength, op, border):
    """one PostChain per stage configuration (the LUT is packed once)"""
    key = (lut, strength, op, border)
    if key not in env["chains"]:
        env["chains"][key] = pkg.chain.PostChain(
            lut=dict(lut_data=env["lut"][lut], strength=strength) if lut else None,
            stencil=dict(op=op, strength=rcm.STRENGTH[op], border=border) if op else None, device=dev)
    return env["chains"][key]


def _oracle_lut(olut, dtype):
    """The table as the reference's VRGDG_LUTS sees it on frames of `dtype`: the node converts DOMAIN_MIN / DOMAIN_MAX to the image
    dtype and takes the span there (VRGDG_IV_Adjustments.py:349-361), then grades in fp32.  Expressed as fp32 bounds for the
    up-cast input (dmin16 + span16 is exact in fp32, so the oracle's span is span16); a unit domain is unchanged."""
    if dtype == "f32":
        return olut
    dmin = olut["domain_min"].to(TORCH[dtype])
    span = torch.clamp(olut["domain_max"].to(TORCH[dtype]) - dmin, min=1e-6)
    return dict(olut, domain_min=dmin.float(), domain_max=dmin.float() + span.float())


def _expected(oracle, env, c, x):
    lut = dict(lut_data=_oracle_lut(env["olut"][c.lut], c.dtype), strength=c.strength) if c.lut else None
    st = dict(op=c.op, border=c.border, strength=rcm.STRENGTH[c.op]) if c.op else None
    return oracle.chain_compose(x.float(), lut=lut, stencil=st)          # 16-bit frames: the oracle on the up-cast input


def _maxdiff(a, b):
    return (a.float().cpu() - b.float().cpu()).abs().max().item()


@pytest.mark.parametrize("c", rcm.CASES, ids=rcm.case_id)
def test_rgba_chain_vs_oracle(pkg, oracle, cuda_device, env, monkeypatch, c):
    nv = pkg._native
    x = _rgba(c.dtype, c.shape)
    chain = _chain(pkg, env, cuda_device, c.lut, c.strength, c.op, c.border)
    if c.shape == "ragged":
        monkeypatch.setenv("VRGDG_NO_TMA", "1")
    got = chain(x.to(cuda_device))
    torch.cuda.synchronize()
    if c.op:
        assert nv.last_tile_path() == rcm.PATH[c.shape]
    assert got.dtype == x.dtype and got.shape == x.shape and got.device == cuda_device
    assert not torch.equal(got.cpu(), x), "an enabled stage left the frames unchanged"
    want = _expected(oracle, env, c, x)
    if c.dtype == "f32":
        assert torch.equal(got.cpu(), want), "max |diff| %.3g, want bit-identical" % _maxdiff(got, want)
    else:
        assert _maxdiff(got, want) <= rcm.ULP[c.dtype]


@pytest.mark.parametrize("shape", ["tma", "ragged"])
@pytest.mark.parametrize("strength", rcm.LUT_STRENGTHS)
@pytest.mark.parametrize("lut", ["vintage33", "domain5"])
@pytest.mark.parametrize("pair", rcm.PAIRS, ids=lambda p: "op%d-border%d" % p)
@pytest.mark.parametrize("dtype", rcm.DTYPES)
def test_rgb_channels_equal_the_three_channel_chain(pkg, cuda_device, env, monkeypatch, dtype, pair, lut, strength, shape):
    x = _rgba(dtype, shape, seed=5).to(cuda_device)
    chain = _chain(pkg, env, cuda_device, lut, strength, *pair)
    if shape == "ragged":
        monkeypatch.setenv("VRGDG_NO_TMA", "1")
    got = chain(x)
    rgb = chain(x[..., :3].contiguous())
    assert torch.equal(got[..., :3], rgb)


@pytest.mark.parametrize("strength", rcm.LUT_STRENGTHS)
@pytest.mark.parametrize("lut", list(rcm.LUTS))
@pytest.mark.parametrize("pair", rcm.PAIRS, ids=lambda p: "op%d-border%d" % p)
def test_fp32_equals_the_two_kernel_composition(pkg, cuda_device, env, pair, lut, strength):
    """one pass = ops.lut3d_apply (k_lut_rgba) then ops.stencil3x3 (k_tile<float, 0, true, 4>), bit for bit"""
    x = _rgba("f32", "tma", seed=9).to(cuda_device)
    chain = _chain(pkg, env, cuda_device, lut, strength, *pair)
    got = chain(x)
    data = env["lut"][lut]
    dmin = data["domain_min"].float()
    span = torch.clamp(data["domain_max"].float() - dmin, min=1e-6)
    blend = strength / 10.0
    lutted = pkg.ops.lut3d_apply(x, chain._luts[cuda_device], dmin.tolist(), span.tolist(), blend, 1.0 - blend)
    two = pkg.ops.stencil3x3(lutted, pair[0], rcm.STRENGTH[pair[0]], pair[1])
    assert torch.equal(got, two)


@pytest.mark.parametrize("dtype", rcm.DTYPES)
def test_tma_equals_generic_loader(pkg, cuda_device, env, monkeypatch, dtype):
    nv = pkg._native
    x = _rgba(dtype, "tma", seed=3).to(cuda_device)
    for op, border in rcm.PAIRS:
        chain = _chain(pkg, env, cuda_device, "vintage33", 3.5, op, border)
        a = chain(x)
        assert nv.last_tile_path() == "tma"
        monkeypatch.setenv("VRGDG_NO_TMA", "1")
        b = chain(x)
        assert nv.last_tile_path() == "generic"
        monkeypatch.delenv("VRGDG_NO_TMA")
        assert torch.equal(a, b), (op, border)


def test_full_hd_rgba_chain_vs_oracle(pkg, oracle, cuda_device, env):
    x = _rgba("f32", (1, 1080, 1920), seed=21)
    chain = _chain(pkg, env, cuda_device, "vintage33", 10.0, 1, 0)
    got = chain(x.to(cuda_device))
    assert pkg._native.last_tile_path() == "tma"
    want = oracle.chain_compose(x, lut=dict(lut_data=env["olut"]["vintage33"], strength=10.0), stencil=dict(op=1, border=0, strength=rcm.STRENGTH[1]))
    assert torch.equal(got.cpu(), want)


def test_rgba_chain_rejections_on_the_device(pkg, cuda_device, env):
    x = _rgba("f32", "small").to(cuda_device)
    d = pkg._native.ChainDesc()
    d.stencil_op = 1
    with pytest.raises(ValueError, match="ext_noise"):
        pkg.ops.chain_apply(x, d, ext_noise=torch.zeros_like(x))
    with pytest.raises(ValueError, match="3 or 4"):
        pkg.ops.chain_apply(x[..., :2].contiguous(), d)
    with pytest.raises(ValueError, match="uint8"):
        pkg.ops.chain_apply((x * 255).to(torch.uint8), d)
    d.stencil_op = 3
    with pytest.raises(ValueError, match="takes 3 channels"):
        pkg.ops.chain_apply(x, d)
    d.stencil_op, d.grain_enabled = 1, 1
    with pytest.raises(ValueError, match="film grain"):
        pkg.ops.chain_apply(x, d)
    # nothing enabled: a copy
    assert torch.equal(pkg.ops.chain_apply(x, pkg._native.ChainDesc()), x)


NODE_CALLS = [("unsharp", False, "FastUnsharpSharpen"), ("unsharp", True, "FastUnsharpSharpen"),
              ("laplacian", False, "FastLaplacianSharpen"), ("sobel", False, "FastSobelSharpen")]


def _node(pkg, images, sharpen, use_gpu, lut_strength=7.5):
    return pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_PostChain"]().apply_chain(images, 0.0, 0.5, 1.0, NODE_LUT, lut_strength, sharpen, 0.4,
                                                                         use_gpu, 3)[0]


def _stock(pkg, images, key, use_gpu, lut_strength=7.5):
    lutted = pkg.VRGDG_LUTS().apply_lut(images, NODE_LUT, "auto", lut_strength)[0]
    node = pkg.NODE_CLASS_MAPPINGS[key]()
    return getattr(node, node.FUNCTION)(lutted, 0.4, use_gpu)[0]


@pytest.mark.parametrize("dtype", rcm.DTYPES)
@pytest.mark.parametrize("where", ["host", "cuda"])
@pytest.mark.parametrize("sharpen, use_gpu, key", NODE_CALLS)
def test_post_chain_node_on_rgba_matches_the_stock_nodes(pkg, cuda_device, where, dtype, sharpen, use_gpu, key):
    """VRGDG_B200_PostChain = VRGDG_LUTS -> Fast*Sharpen on an RGBA batch, result where the input was.  fp32: bit for bit.  16-bit:
    within one spacing of the stock nodes run on the up-cast batch (the stock pair rounds the LUT result to 16 bits in between,
    the fused pass does not)"""
    x = _rgba(dtype, (5, 48, 96), seed=13)
    src = x if where == "host" else x.to(cuda_device)
    got = _node(pkg, src, sharpen, use_gpu)
    assert got.device == src.device and got.shape == x.shape and got.dtype == x.dtype
    up = x.float() if where == "host" else x.float().to(cuda_device)
    want = _stock(pkg, up, key, use_gpu)
    if dtype == "f32":
        assert torch.equal(got.cpu(), want.cpu())
    else:
        assert _maxdiff(got, want) <= rcm.ULP[dtype]


@pytest.mark.parametrize("sharpen, use_gpu, key", NODE_CALLS)
def test_sharded_rgba_chain_matches_the_unsharded_node(pkg, cuda_device, monkeypatch, sharpen, use_gpu, key):
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    x = _rgba("f32", (7, 48, 96), seed=11)
    one = _node(pkg, x, sharpen, use_gpu)
    rt = importlib.import_module(pkg.__name__ + "._runtime")
    seen = []
    sharded = rt.stream_frames_sharded

    def traced(src, make_fn, chunk, out_device, devs, out=None):
        seen.append([torch.device(d) for d in devs])
        return sharded(src, make_fn, chunk, out_device, devs, out=out)
    monkeypatch.setattr(rt, "stream_frames_sharded", traced)
    monkeypatch.setattr(importlib.import_module(pkg.__name__ + ".chain_nodes"), "devices_from_env", lambda: [cuda_device, cuda_device])
    got = _node(pkg, x, sharpen, use_gpu)
    assert seen == [[cuda_device, cuda_device]]
    assert got.device.type == "cpu" and got.shape == x.shape and not torch.equal(got, x)
    assert torch.equal(got, one)

"""RGBA IMAGE batches through the 3x3 sharpeners (k_tile with CH = 4, vrgdg_stencil3x3_ch) against the oracle, channel by channel
against the 3-channel kernel, and through the nodes: host and CUDA batches, the VRGDG_LUTS -> FastUnsharpSharpen graph, sharding.
The cases come from tests/rgba_stencil_matrix.py, whose CPU guard checks that they reach every launch_tile_rgba path."""
import importlib
import os

import pytest
import torch

import rgba_stencil_matrix as rsm
from helpers import LUTS, natural_frames

pytestmark = pytest.mark.gpu

TORCH = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
LUT = "B200 Vintage 33.cube"


def _reference(oracle, op, border):
    return {(rsm.BOX_UNSHARP, rsm.REPLICATE): oracle.unsharp_numpy, (rsm.BOX_UNSHARP, rsm.ZERO): oracle.unsharp_torch,
            (rsm.LAPLACIAN_CPU, rsm.REPLICATE): oracle.laplacian_numpy, (rsm.SOBEL_CPU, rsm.REPLICATE): oracle.sobel_numpy}[(op, border)]


def _rgba(B, H, W, seed, dtype=torch.float32):
    """natural RGB frames and a spatially coherent alpha plane of its own (an edge-free alpha would hide a wrong neighbour)"""
    alpha = natural_frames(B, H, W, seed=seed + 1000)[..., 1:2]
    return torch.cat([natural_frames(B, H, W, seed=seed), alpha], dim=-1).contiguous().to(dtype)


def _maxdiff(a, b):
    return (a.float().cpu() - b.float().cpu()).abs().max().item()


def _cards():
    return [torch.device("cuda", i) for i in range(torch.cuda.device_count()) if tuple(torch.cuda.get_device_capability(i)) == (9, 0)]


@pytest.mark.parametrize("case", rsm.CASES, ids=lambda c: "%s-op%d-border%d-%s" % (c.dtype, c.op, c.border, c.shape))
def test_rgba_stencil_vs_oracle(pkg, oracle, cuda_device, monkeypatch, case):
    nv = pkg._native
    B, H, W = rsm.SHAPES[case.shape]
    x = _rgba(B, H, W, seed=H * W + case.op, dtype=TORCH[case.dtype])
    s = rsm.STRENGTH[case.op]
    if case.shape == "ragged":
        monkeypatch.setenv("VRGDG_NO_TMA", "1")
    got = pkg.ops.stencil3x3(x.to(cuda_device), case.op, s, case.border)
    assert nv.last_tile_path() == rsm.PATH[case.shape]
    assert got.dtype == x.dtype and got.shape == x.shape
    want = _reference(oracle, case.op, case.border)(x.float(), s)          # 16-bit frames: the oracle on the up-cast input
    if case.dtype == "f32":
        assert torch.equal(got.cpu(), want)
    else:
        assert _maxdiff(got, want) <= rsm.ULP[case.dtype]


@pytest.mark.parametrize("shape", ["tma", "ragged"])
@pytest.mark.parametrize("border", [rsm.REPLICATE, rsm.ZERO])
@pytest.mark.parametrize("op", rsm.RGBA_OPS)
@pytest.mark.parametrize("dtype", rsm.DTYPES)
def test_each_channel_equals_the_three_channel_kernel(pkg, cuda_device, dtype, op, border, shape):
    """RGB of the RGBA result = the 3-channel kernel on the RGB planes; alpha = the 3-channel kernel on alpha in all three channels"""
    B, H, W = rsm.SHAPES[shape]
    x = _rgba(B, H, W, seed=7 + op, dtype=TORCH[dtype]).to(cuda_device)
    s = rsm.STRENGTH[op]
    got = pkg.ops.stencil3x3(x, op, s, border)
    rgb = pkg.ops.stencil3x3(x[..., :3].contiguous(), op, s, border)
    alpha = pkg.ops.stencil3x3(x[..., 3:4].expand(-1, -1, -1, 3).contiguous(), op, s, border)
    assert torch.equal(got[..., :3], rgb)
    assert torch.equal(got[..., 3], alpha[..., 0])
    assert not torch.equal(got, x)


@pytest.mark.parametrize("dtype", rsm.DTYPES)
def test_tma_equals_generic_loader(pkg, cuda_device, monkeypatch, dtype):
    nv = pkg._native
    x = _rgba(*rsm.SHAPES["tma"], seed=3, dtype=TORCH[dtype]).to(cuda_device)
    for op in rsm.RGBA_OPS:
        for border in (rsm.REPLICATE, rsm.ZERO):
            a = pkg.ops.stencil3x3(x, op, 0.6, border)
            assert nv.last_tile_path() == "tma"
            monkeypatch.setenv("VRGDG_NO_TMA", "1")
            b = pkg.ops.stencil3x3(x, op, 0.6, border)
            assert nv.last_tile_path() == "generic"
            monkeypatch.delenv("VRGDG_NO_TMA")
            assert torch.equal(a, b), (op, border)


def test_full_hd_rgba_unsharp_vs_oracle(pkg, oracle, cuda_device):
    x = _rgba(1, 1080, 1920, seed=21)
    got = pkg.ops.stencil3x3(x.to(cuda_device), rsm.BOX_UNSHARP, 0.5, rsm.REPLICATE)
    assert pkg._native.last_tile_path() == "tma"
    assert torch.equal(got.cpu(), oracle.unsharp_numpy(x, 0.5))


def test_rgba_rejections_on_the_device(pkg, cuda_device):
    nv = pkg._native
    x = _rgba(1, 40, 80, seed=1).to(cuda_device)
    for op in (rsm.LAPLACIAN_GPU, rsm.SOBEL_GPU):
        with pytest.raises(ValueError, match="takes 3 channels"):
            pkg.ops.stencil3x3(x, op, 0.5, rsm.ZERO)
    with pytest.raises(ValueError, match="uint8"):
        pkg.ops.stencil3x3((x * 255).to(torch.uint8), rsm.BOX_UNSHARP, 0.5)
    with pytest.raises(ValueError):
        pkg.ops.stencil3x3(x[..., :2].contiguous(), rsm.BOX_UNSHARP, 0.5)
    assert nv.last_tile_path() in ("tma", "generic")


@pytest.mark.parametrize("use_gpu", [False, True], ids=["numpy_path", "torch_path"])
@pytest.mark.parametrize("where", ["host", "cuda"])
def test_lut_then_unsharp_graph_on_rgba(pkg, oracle, cuda_device, where, use_gpu):
    """VRGDG_LUTS -> FastUnsharpSharpen on an RGBA batch: the reference's composition, bit for bit (fp32), result where the input was"""
    x = _rgba(3, 48, 96, seed=5)
    src = x if where == "host" else x.to(cuda_device)
    lutted = pkg.VRGDG_LUTS().apply_lut(src, LUT, "auto", 7.5)[0]
    out = pkg.FastUnsharpSharpen().apply_unsharp(lutted, 0.5, use_gpu)[0]
    sharpen = oracle.unsharp_torch if use_gpu else oracle.unsharp_numpy
    want = sharpen(oracle.apply_lut(x, oracle.parse_cube(os.path.join(LUTS, LUT)), 7.5), 0.5)
    assert out.device == src.device and out.shape == x.shape
    assert torch.equal(out.cpu(), want)
    vt = importlib.import_module(pkg.__name__ + ".video_tools")              # the enhancer's helper takes RGBA through the same op
    assert torch.equal(vt._apply_unsharp(lutted, 0.5, use_gpu).cpu(), want)


@pytest.mark.parametrize("key, use_gpu", [("FastLaplacianSharpen", False), ("FastSobelSharpen", False)])
def test_laplacian_and_sobel_nodes_on_rgba(pkg, oracle, cuda_device, key, use_gpu):
    x = _rgba(2, 40, 72, seed=9)
    node = pkg.NODE_CLASS_MAPPINGS[key]()
    for src in (x, x.to(cuda_device)):
        out = getattr(node, node.FUNCTION)(src, 0.4, use_gpu)[0]
        want = (oracle.laplacian_numpy if key == "FastLaplacianSharpen" else oracle.sobel_numpy)(x, 0.4)
        assert out.device == src.device and torch.equal(out.cpu(), want)
    for half in (torch.float16, torch.bfloat16):
        out = getattr(node, node.FUNCTION)(x.to(half), 0.4, use_gpu)[0]
        assert out.dtype == half


NODE_CALLS = [("FastUnsharpSharpen", False), ("FastUnsharpSharpen", True), ("FastLaplacianSharpen", False), ("FastSobelSharpen", False)]


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("devices", ["two_workers_one_card", "every_card"])
@pytest.mark.parametrize("key, use_gpu", NODE_CALLS)
def test_sharded_rgba_batch_matches_the_unsharded_node(pkg, cuda_device, monkeypatch, key, use_gpu, devices, pinned):
    cards = [cuda_device] * 2 if devices == "two_workers_one_card" else _cards()
    if len(cards) < 2:
        pytest.skip("one compute-capability-9.0 device visible; the two-worker case covers the sharded path")
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    x = _rgba(7, 48, 96, seed=11)
    x = x.pin_memory() if pinned else x
    monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(2 * x[0].numel() * x.element_size()))     # 2-frame chunks
    node = pkg.NODE_CLASS_MAPPINGS[key]()
    run = lambda: getattr(node, node.FUNCTION)(x, 0.5, use_gpu)[0]
    one = run()
    rt = importlib.import_module(pkg.__name__ + "._runtime")
    seen = []
    sharded = rt.stream_frames_sharded

    def traced(src, make_fn, chunk, out_device, devs, out=None):
        seen.append([torch.device(d) for d in devs])
        return sharded(src, make_fn, chunk, out_device, devs, out=out)
    monkeypatch.setattr(rt, "stream_frames_sharded", traced)
    monkeypatch.setattr(importlib.import_module(pkg.__name__ + ".filter_nodes"), "devices_from_env", lambda: list(cards))
    got = run()
    assert seen == [cards]
    assert got.device.type == "cpu" and got.shape == x.shape and not torch.equal(one, x)
    assert torch.equal(got, one)


def test_other_frame_nodes_still_refuse_rgba(pkg, cuda_device):
    x = _rgba(1, 16, 16, seed=2)
    with pytest.raises(ValueError):
        pkg.FastFilmGrain().apply_grain(x, 0.04, 0.5, 4)
    with pytest.raises(ValueError):
        pkg.ColorMatchToReference().match_color(x, x[..., :3].contiguous(), 1.0, 1)
    with pytest.raises(ValueError):
        pkg.ColorMatchToReference().match_color(x[..., :3].contiguous(), x, 1.0, 1)

"""Torch-stream grain on the GPU: the in-kernel draws equal torch.randn of fresh seeded CUDA generators bit for bit (sign of zero
included), and the grain helpers / the EnhanceFrames node with noise="torch_cuda" equal the reference run on CUDA tensors.  The
defaults ("vrgdg") keep this package's own generator."""
import importlib

import numpy as np
import pytest
import torch

from helpers import natural_frames

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1), (17, 23), (64, 64), (1080, 1920), (2160, 3840)]
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
INT_VIEW = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}


def _vt(pkg):
    return importlib.import_module(pkg.__name__ + ".video_tools")


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _per_frame_draws(B, H, W, seed, frame0, dtype):
    return torch.stack([torch.randn([H, W, 3], generator=_gen((seed + frame0 + i) & 0x7FFFFFFF), device="cuda", dtype=dtype)
                        for i in range(B)])


def _bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(INT_VIEW[a.dtype]), b.view(INT_VIEW[b.dtype]))


def _within_one_spacing(a, b):
    """16-bit frames in [0, 1]: neighbouring values of the dtype differ by one in their bit patterns"""
    ia, ib = a.view(torch.int16).to(torch.int32), b.view(torch.int16).to(torch.int32)
    return bool(((a == b) | ((ia - ib).abs() <= 1)).all())


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dx%d" % s)
def test_per_frame_stream_is_torch_randn(pkg, cuda_device, shape, dtype):
    H, W = shape
    B = 1 if H * W > 1920 * 1080 else 2
    for seed in (0, 42, 0x7FFFFFFF):
        for frame0 in (0, 10**6):
            got = pkg.ops.grain_noise(B, H, W, seed, frame0, pkg._native.SEED_TORCH_PER_FRAME).to(dtype)
            assert _bits_equal(got, _per_frame_draws(B, H, W, seed, frame0, dtype)), (seed, frame0)


@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_per_call_stream_is_one_torch_randn(pkg, cuda_device, B, dtype):
    H, W = (1080, 1920) if B == 8 else (61, 97)
    for seed in (-1, 2**63, 5):
        got = pkg.ops.grain_noise(B, H, W, seed, 123, pkg._native.SEED_TORCH_PER_CALL).to(dtype)
        want = torch.randn([B, H, W, 3], generator=_gen(seed), device="cuda", dtype=dtype)
        assert _bits_equal(got, want), seed


def test_stream_holds_positive_zeros_where_u_rounds_to_one(pkg, cuda_device):
    """u = a 2^-32 + 2^-33 rounds to 1.0f for the top 2^-24 of words: radius -0 * sin, which ATen's z * 1 + 0 makes +0.  A 4K draw
    holds a few of them; they must come out as +0, as torch's do."""
    got = pkg.ops.grain_noise(1, 2160, 3840, 9, 0, pkg._native.SEED_TORCH_PER_FRAME)
    want = _per_frame_draws(1, 2160, 3840, 9, 0, torch.float32)
    assert _bits_equal(got, want)
    assert not bool(torch.signbit(got[got == 0]).any())


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_film_grain_tensor_matches_the_reference_on_cuda(pkg, oracle, cuda_device, dtype):
    vt = _vt(pkg)
    x = natural_frames(3, 45, 67, seed=4).to("cuda", dtype)
    for seed in (7, 2**40 + 3):
        got = vt._apply_film_grain_tensor(x, 0.3, 0.4, "cuda", seed, noise="torch_cuda")
        assert got.device == x.device
        if dtype == torch.float32:
            assert torch.equal(got, oracle.film_grain_tensor(x, 0.3, 0.4, seed))
        else:
            # the project's 16-bit rule: the oracle on the up-cast input (here with the reference's 16-bit draw, up-cast), rounded once
            z = torch.randn(x.shape, dtype=dtype, device="cuda", generator=_gen(seed)).float()
            want = (x.float() + oracle.grain_mix(z, 0.4) * 0.3).clamp(0.0, 1.0).to(dtype)
            assert _within_one_spacing(got, want)


def _seeded_grain_reference(oracle, x, intensity, sat, seed, frame_start):
    """_apply_seeded_grain on a CUDA tensor: a per-frame CUDA generator, grain_mix, x + mixed * I, clamp"""
    z = _per_frame_draws(x.shape[0], x.shape[1], x.shape[2], seed, frame_start, x.dtype)
    mixed = torch.stack([oracle.grain_mix(f, sat) for f in z], dim=0)
    return (x + mixed * intensity).clamp(0.0, 1.0)


@pytest.mark.parametrize("shape", [(33, 47), (64, 64), (1080, 1920)], ids=lambda s: "%dx%d" % s)
def test_seeded_grain_matches_the_reference_on_cuda(pkg, oracle, cuda_device, shape):
    x = natural_frames(3, *shape, seed=5).cuda()
    for seed, frame_start in ((42, 0), (0x7FFFFFFF, 10**6), (123, 7)):
        got = _vt(pkg)._apply_seeded_grain(x, 0.06, 0.35, seed, frame_start, noise="torch_cuda")
        assert torch.equal(got, _seeded_grain_reference(oracle, x, 0.06, 0.35, seed, frame_start))


def test_seeded_grain_batch_boundaries(pkg, cuda_device):
    """the reference's own batch-boundary check: frames [0:4] at frame_start 100 = [0:2] at 100 followed by [2:4] at 102"""
    sg = _vt(pkg)._apply_seeded_grain
    x = natural_frames(4, 40, 52, seed=6).cuda()
    whole = sg(x, 0.05, 0.5, 11, 100, noise="torch_cuda")
    parts = torch.cat([sg(x[0:2], 0.05, 0.5, 11, 100, noise="torch_cuda"), sg(x[2:4], 0.05, 0.5, 11, 102, noise="torch_cuda")])
    assert torch.equal(whole, parts)


def _settings(use_gpu, sharpen=0.7, grain=0.05):
    return dict(use_gpu=use_gpu, sharpen_enabled=sharpen > 0, sharpen_strength=sharpen, grain_enabled=grain > 0, grain_intensity=grain,
                saturation_mix=0.4, seed=31)


@pytest.mark.parametrize("use_gpu", [True, False])
@pytest.mark.parametrize("shape", [(37, 53), (270, 480)], ids=lambda s: "%dx%d" % s)
def test_fused_effects_equal_the_two_helpers(pkg, cuda_device, use_gpu, shape):
    vt = _vt(pkg)
    x = natural_frames(3, *shape, seed=8).cuda()
    st = _settings(use_gpu)
    want = vt._apply_seeded_grain(vt._apply_unsharp(x, 0.7, use_gpu), 0.05, 0.4, 31, 9, noise="torch_cuda").cpu()
    assert torch.equal(vt._apply_effects_batch(x, st, 9, noise="torch_cuda"), want)
    node = pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_EnhanceFrames"]()
    assert torch.equal(node.enhance(x, 0.7, 0.05, 0.4, 31, 9, use_gpu, noise_stream="torch_cuda")[0].cpu(), want)
    # grain alone (no sharpen) takes vrgdg_grain
    only = vt._apply_effects_batch(x, _settings(use_gpu, sharpen=0.0), 9, noise="torch_cuda")
    assert torch.equal(only, vt._apply_seeded_grain(x, 0.05, 0.4, 31, 9, noise="torch_cuda").cpu())


def test_enhance_frames_bytes_match_the_reference_on_cuda(pkg, oracle, cuda_device):
    """uint8 frames through resize -> unsharp -> per-frame CUDA grain -> bytes, against the reference's helpers run on CUDA: Lanczos4
    (bit-exact oracle), _frames_to_tensor, the use_gpu unsharp (avg_pool2d on CUDA), the CUDA draws, _tensor_to_frames."""
    vt = _vt(pkg)
    rng = np.random.default_rng(3)
    frames = [rng.integers(0, 256, (48, 64, 3), dtype=np.uint8) for _ in range(3)]
    st = _settings(True)
    got = vt.enhance_frames(frames, 80, 60, st, frame_start=5, noise="torch_cuda")
    x = oracle.frames_to_tensor(oracle.resize_frames(frames, 80, 60)).cuda()
    sharp = oracle.unsharp_torch(x, 0.7)
    ours_sharp = vt._apply_unsharp(x, 0.7, True)
    diff = (sharp != ours_sharp)
    if bool(diff.any()):     # CUDA avg_pool2d is not pinned to the kernel: grain alone is pinned behind the package's unsharp
        print("CUDA avg_pool2d vs the unsharp kernel: %d of %d elements differ, max |diff| %.3g"
              % (int(diff.sum()), diff.numel(), float((sharp - ours_sharp).abs().max())))
        sharp = ours_sharp
    want = oracle.tensor_to_frames(_seeded_grain_reference(oracle, sharp, 0.05, 0.4, 31, 5))
    assert len(got) == 3
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


def test_enhance_frames_node_sharded_over_two_workers_on_one_card(pkg, monkeypatch, cuda_device):
    x = natural_frames(6, 72, 96, seed=9)                       # host batch: the node shards it over VRGDG_DEVICES
    node = pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_EnhanceFrames"]()
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    one = node.enhance(x, 0.6, 0.05, 0.3, 42, 3, True, noise_stream="torch_cuda")[0]
    mod = importlib.import_module(pkg.__name__ + ".chain_nodes")
    monkeypatch.setattr(mod, "devices_from_env", lambda: [torch.device("cuda", 0), torch.device("cuda", 0)])
    two = node.enhance(x, 0.6, 0.05, 0.3, 42, 3, True, noise_stream="torch_cuda")[0]
    assert torch.equal(one, two)
    two_grain_only = node.enhance(x, 0.0, 0.05, 0.3, 42, 3, True, noise_stream="torch_cuda")[0]
    monkeypatch.setattr(mod, "devices_from_env", lambda: None)
    assert torch.equal(two_grain_only, node.enhance(x, 0.0, 0.05, 0.3, 42, 3, True, noise_stream="torch_cuda")[0])


def test_post_chain_post_grain_in_torch_mode(pkg, oracle, cuda_device):
    """PostChain(post_grain=dict(seed_mode=SEED_TORCH_PER_FRAME)) on uint8 and fp32 frames = unsharp then the CUDA draws"""
    nv, vt = pkg._native, _vt(pkg)
    x = natural_frames(2, 50, 70, seed=10).cuda()
    post = dict(intensity=0.05, saturation_mix=0.4, seed=31, seed_mode=nv.SEED_TORCH_PER_FRAME)
    for border, use_gpu in ((nv.BORDER_ZERO, True), (nv.BORDER_REPLICATE, False)):
        chain = pkg.chain.PostChain(stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.7, border=border), post_grain=post)
        want = _seeded_grain_reference(oracle, vt._apply_unsharp(x, 0.7, use_gpu), 0.05, 0.4, 31, 4)
        assert torch.equal(chain(x, first_frame=4), want)
        u8 = pkg.ops.rgb_to_u8bgr(x)
        got = chain(u8, first_frame=4)
        want8 = pkg.ops.rgb_to_u8bgr(_seeded_grain_reference(oracle, vt._apply_unsharp(pkg.ops.u8bgr_to_rgb(u8), 0.7, use_gpu), 0.05, 0.4, 31, 4))
        assert torch.equal(got, want8)


def test_defaults_keep_the_package_generator(pkg, cuda_device):
    """without `noise` the helpers run the package's own PER_CLIP / PER_FRAME generator exactly as before"""
    nv, vt, ops = pkg._native, _vt(pkg), pkg.ops
    x = natural_frames(3, 40, 56, seed=12).cuda()
    assert torch.equal(vt._apply_film_grain_tensor(x, 0.2, 0.5, "cuda", 9), ops.grain(x, 0.2, 0.5, 0.5, 9, 0, nv.SEED_PER_CLIP))
    assert torch.equal(vt._apply_seeded_grain(x, 0.2, 0.5, 9, 4), ops.grain(x, 0.2, 0.5, 0.5, 9, 4, nv.SEED_PER_FRAME))
    st = _settings(True)
    fused = vt._apply_effects_batch(x, st, 4)
    assert torch.equal(fused, vt._apply_effects_batch(x, st, 4, noise="vrgdg"))
    chain = pkg.chain.PostChain(stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.7, border=nv.BORDER_ZERO),
                                post_grain=dict(intensity=0.05, saturation_mix=0.4, seed=31, seed_mode=nv.SEED_PER_FRAME))
    assert torch.equal(fused, chain(x, first_frame=4).cpu())
    node = pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_EnhanceFrames"]()
    assert torch.equal(node.enhance(x, 0.7, 0.05, 0.4, 31, 4, True)[0].cpu(), fused)
    assert not torch.equal(fused, vt._apply_effects_batch(x, st, 4, noise="torch_cuda"))

"""The adjust, resample, blend, 4-channel LUT and uint8 codec kernels on every frame dtype they are built for, against the oracle
(not against other kernels).

The matrix (tests/video_tools_matrix.py): adjust in seven settings x fp32 / fp16 / bf16 / uint8 x shapes that select every clarity
window (K = 1, 3, 5, 7, 9) with the small side as H and as W, on the vector (W % 4 == 0) and scalar stores, and multi-tile frames
whose last tile is partial both ways; resize in all four modes x fp32 / fp16 / bf16 x 3 and 4 channels x stretch, crop to fill,
letterbox, the letterbox restore ROI and an inner ROI, plus one-axis strips whose area windows have products o*in past 2^24; blend,
the 4-channel LUT and the codecs on every float dtype; and one uint8 LUT stream past the 2^30-pixel launch split.

16-bit frames are compared with the oracle run on the up-cast fp32 input and rounded once to the frame dtype; uint8 frames with
oracle.frames_to_tensor -> op -> oracle.tensor_to_frames.  Error bars: video_tools_matrix (resize_bar; every other case is equal)."""
import functools
import importlib
import os

import numpy as np
import pytest
import torch

import video_tools_matrix as vtm
from helpers import LUTS, natural_frames

pytestmark = pytest.mark.gpu

DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16, "u8": torch.uint8}
BITS = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}
LUT_FILE = os.path.join(LUTS, "B200 Vintage 33.cube")
PKG = "comfyui-vrgamedevgirl_b200"
_TORCH_SQRT = torch.sqrt


def _sqrt_rn(x):
    """correctly rounded square root (the float64 root of the fp32 argument, rounded once), like the kernel's __fsqrt_rn; torch's CPU
    sqrt is MKL's < 1 ulp routine"""
    return _TORCH_SQRT(x.double()).to(x.dtype)


def _diff(got, want):
    d = (got.double() - want.double()).abs()
    return "max |diff| %.3g on %d of %d elements" % (float(d.max()), int((got != want).sum()), got.numel())


def _same(got, want):
    assert got.dtype == want.dtype and got.shape == want.shape
    assert torch.equal(got, want), _diff(got, want)


# ---- adjust -----------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _adjust_frames(dtype, shape):
    B, H, W = vtm.ADJUST_SHAPES[shape]
    x = natural_frames(B, H, W, seed=H * 1000 + W) * 1.2 - 0.1          # outside [0, 1]: the source clamp is part of the op
    if dtype == "u8":
        return (x.clamp(0, 1) * 255).round().to(torch.uint8)              # BGR bytes
    return x.to(DT[dtype])


def _adjust_expected(oracle, monkeypatch, c, x):
    st = vtm.ADJUST_SETTINGS[c.setting]
    with monkeypatch.context() as m:
        m.setattr(torch, "sqrt", _sqrt_rn)
        if c.dtype == "u8":
            return torch.from_numpy(oracle.tensor_to_frames(oracle.adjust(oracle.frames_to_tensor(x.numpy()), st)))
        return oracle.adjust(x.float(), st).to(x.dtype)


@pytest.mark.parametrize("c", vtm.ADJUST_CASES, ids=vtm.adjust_id)
def test_adjust_vs_oracle(pkg, oracle, cuda_device, monkeypatch, c):
    vt = importlib.import_module(PKG + ".video_tools")
    x = _adjust_frames(c.dtype, c.shape)
    B, H, W = vtm.ADJUST_SHAPES[c.shape]
    desc = vt._adjust_desc(vtm.ADJUST_SETTINGS[c.setting], H, W)
    assert desc.blur_kernel == vtm.blur_kernel(H, W)
    before = pkg._native.launch_count()
    out = pkg.ops.adjust(x.to(cuda_device), desc)
    torch.cuda.synchronize()
    assert pkg._native.launch_count() - before == len(vtm.adjust_kernels(c))    # point pass + one per box pass of the mirror
    assert out.dtype == x.dtype and out.shape == x.shape and out.device == cuda_device
    _same(out.cpu(), _adjust_expected(oracle, monkeypatch, c, x))


# ---- resize -----------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _resize_frames(dtype, channels, geometry):
    B, H, W = (2, 80, 80) if geometry == "restore" else vtm.RESIZE_SRC
    x = natural_frames(B, H, W, seed=H * 100 + W + channels) * 1.2 - 0.1
    if channels == 4:
        x = torch.cat([x, torch.rand(B, H, W, 1, generator=torch.Generator().manual_seed(W))], dim=-1)
    return x.to(DT[dtype])


@functools.lru_cache(maxsize=None)
def _strip(dtype, axis, n_in):
    """a [1, 2, n_in + 1, 3] (x) or [1, n_in + 1, 2, 3] (y) strip; the ROI leaves out the last column / row, which holds 1.0"""
    g = torch.Generator().manual_seed(n_in)
    if axis == "x":
        x = torch.rand(1, 2, n_in + 1, 3, generator=g)
        x[:, :, -1] = 1.0
    else:
        x = torch.rand(1, n_in + 1, 2, 3, generator=g)
        x[:, -1] = 1.0
    return x.to(DT[dtype])


def _run_resize(pkg, oracle, c, dev):
    """(kernel result on the device, oracle result rounded to the frame dtype)"""
    ve = importlib.import_module(PKG + ".video_enhance")
    method = vtm.METHOD[c.mode]
    strip = vtm.strip_of(c)
    if strip:
        axis, n_in, n_out = strip
        x = _strip(c.dtype, axis, n_in)
        sw, sh, rw, rh = (n_in, 2, n_out, 2) if axis == "x" else (2, n_in, 2, n_out)
        got = pkg.ops.resize(x.to(dev), rh, rw, c.mode, roi=(0, 0, sw, sh), resampled=(rw, rh))
        want = oracle.resize_batch(x[:, :sh, :sw].float(), rw, rh, "Stretch to dimensions", method)
        return got, want.to(x.dtype)
    x = _resize_frames(c.dtype, c.channels, c.geometry)
    fit, tw, th = vtm.RESIZE_GEOMETRIES[c.geometry]
    if c.geometry == "restore":
        got = ve._restore_batch(x.to(dev), tw, th, fit, method)
        want = oracle.restore_batch(x.float(), tw, th, fit, method)
    elif c.geometry == "roi":
        x0, y0, w, h = vtm.ROI
        got = pkg.ops.resize(x.to(dev), th, tw, c.mode, roi=vtm.ROI, resampled=(tw, th))
        want = oracle.resize_batch(x[:, y0:y0 + h, x0:x0 + w].float(), tw, th, fit, method)
    else:
        got = ve._resize_batch(x.to(dev), tw, th, fit, method)
        want = oracle.resize_batch(x.float(), tw, th, fit, method)
    return got, want.to(x.dtype)


@pytest.mark.parametrize("c", vtm.RESIZE_CASES, ids=vtm.resize_id)
def test_resize_vs_oracle(pkg, oracle, cuda_device, c):
    got, want = _run_resize(pkg, oracle, c, cuda_device)
    assert got.dtype == DT[c.dtype] and got.device == cuda_device and got.shape == want.shape
    got = got.cpu()
    bar = vtm.resize_bar(c)
    if bar == 0:
        _same(got, want)
    else:
        err = float((got.double() - want.double()).abs().max())
        assert err <= bar, (err, bar)


# ---- blend ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", vtm.BLEND_CASES, ids=lambda c: "blend-%s-%s" % (c.dtype, c.weights))
def test_blend_vs_oracle(pkg, oracle, cuda_device, c):
    dt = DT[c.dtype]
    B, H, W, C = vtm.BLEND_SHAPE
    orig = (natural_frames(B, H, W, seed=71) * 1.6 - 0.3).to(dt)           # outside [0, 1]
    restored = (natural_frames(B, H, W, seed=72) * 1.6 - 0.3).to(dt)
    s = vtm.BLEND_WEIGHTS[c.weights]
    got = pkg.ops.blend(orig.to(cuda_device), restored.to(cuda_device), 1.0 - s, s)    # (1 - s) formed in Python double
    assert got.dtype == dt and got.shape == orig.shape and got.device == cuda_device
    _same(got.cpu(), oracle.restore_blend(orig.float(), restored.float(), s).to(dt))


# ---- 4-channel LUT ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", vtm.LUT_RGBA_CASES, ids=lambda c: "lut_rgba-%s-%s" % (c.dtype, c.strength))
def test_lut_rgba_vs_oracle(pkg, oracle, cuda_device, c):
    dt = DT[c.dtype]
    olut = dict(oracle.parse_cube(LUT_FILE))
    olut["domain_min"], olut["domain_max"] = (torch.tensor(v, dtype=torch.float32) for v in vtm.LUT_DOMAIN)
    x = natural_frames(2, 37, 53, seed=44) * 1.4 - 0.2
    alpha = torch.rand(2, 37, 53, 1, generator=torch.Generator().manual_seed(45)) * 1.2 - 0.1
    x4 = torch.cat([x, alpha], dim=-1).to(dt)
    strength = vtm.LUT_STRENGTHS[c.strength]
    blend = strength / 10.0
    span = torch.clamp(olut["domain_max"] - olut["domain_min"], min=1e-6)
    got = pkg.ops.lut3d_apply(x4.to(cuda_device), olut["lut"].to(cuda_device), olut["domain_min"].tolist(), span.tolist(), blend, 1.0 - blend)
    assert got.dtype == dt and got.shape == x4.shape and got.device == cuda_device
    got = got.cpu()
    _same(got, oracle.apply_lut(x4.float(), olut, strength).to(dt))
    if blend == 1.0:
        assert torch.equal(got[..., 3].contiguous().view(BITS[dt]), x4[..., 3].contiguous().view(BITS[dt]))    # alpha bit for bit


# ---- codecs -----------------------------------------------------------------------------------------------------------------
def _codec_values(dt):
    """every k/255 in the dtype, both neighbours of each, and values outside [0, 1]"""
    v = (torch.arange(256, dtype=torch.float64) / 255.0).to(dt)
    bits = v.contiguous().view(BITS[dt])
    lowest_negative = torch.iinfo(BITS[dt]).min + 1                       # -(smallest subnormal): the neighbour below +0
    up = (bits + 1).view(dt)
    down = torch.where(bits > 0, bits - 1, torch.full_like(bits, lowest_negative)).view(dt)
    out = torch.cat([v, up, down, torch.tensor([-1e4, -2.0, -0.5, -1e-3, -0.0, 1.5, 2.0, 255.0, 1e4, float("inf"), float("-inf")]).to(dt)])
    pad = (-out.numel()) % 3
    return torch.cat([out, out[:pad]]).view(1, 1, -1, 3)


@pytest.mark.parametrize("c", vtm.CODEC_CASES, ids=lambda c: "codec-%s-%s" % (c.dtype, c.direction))
def test_codecs_vs_oracle(pkg, oracle, cuda_device, c):
    dt = DT[c.dtype]
    if c.direction == "to_float":
        k = torch.arange(256)
        bgr = torch.stack([k, 255 - k, (k * 37 + 11) % 256], dim=-1).to(torch.uint8).view(1, 1, 256, 3)   # every byte in every channel
        got = pkg.ops.u8bgr_to_rgb(bgr.to(cuda_device), dt)
        assert got.dtype == dt and got.shape == bgr.shape and got.device == cuda_device
        _same(got.cpu(), oracle.frames_to_tensor(bgr.numpy()).to(dt))
    else:
        x = _codec_values(dt)
        got = pkg.ops.rgb_to_u8bgr(x.to(cuda_device))
        assert got.dtype == torch.uint8 and got.shape == x.shape and got.device == cuda_device
        want = oracle.tensor_to_frames(x.float())
        got = got.cpu().numpy()
        assert np.array_equal(got, want), "%d of %d bytes differ" % (int((got != want).sum()), got.size)


# ---- the LUT pixel stream past 2^30 pixels ------------------------------------------------------------------------------------
def test_lut_stream_past_2_30_pixels(pkg, oracle, cuda_device):
    """one uint8 stream of 2^30 + 4097 pixels (3.2 GB in, 3.2 GB out): vrgdg_lut3d_apply splits it into a 2^30-pixel launch and an
    odd 4097-pixel one; the lookup is per pixel, so around the split and in the tail the result equals the lookup of small slices"""
    olut = oracle.parse_cube(LUT_FILE)
    n, C = vtm.LUT_STREAM_PIXELS, vtm.LUT_STREAM_CHUNK
    packed = pkg.ops.pack_lut(olut["lut"], cuda_device)
    x = out = None
    try:
        x = torch.empty((1, 1, n, 3), dtype=torch.uint8, device=cuda_device)
        x.random_(0, 256, generator=torch.Generator(device=cuda_device).manual_seed(30))
        out = pkg.ops.lut3d_apply(x, packed, [0.0] * 3, [1.0] * 3, 1.0, 0.0)
        assert out.shape == x.shape and out.dtype == torch.uint8
        for a, b in ((0, 4096), (C - 4096, C + 4096), (n - 8193, n)):
            part = pkg.ops.lut3d_apply(x[:, :, a:b].contiguous(), packed, [0.0] * 3, [1.0] * 3, 1.0, 0.0)
            assert torch.equal(out[:, :, a:b], part), (a, b)
        a, b = C - 4096, C + 4096
        want = oracle.tensor_to_frames(oracle.apply_lut(oracle.frames_to_tensor(x[:, :, a:b].cpu().numpy()), olut, 10.0))
        assert np.array_equal(out[:, :, a:b].cpu().numpy(), want)
    finally:
        del x, out
        torch.cuda.empty_cache()

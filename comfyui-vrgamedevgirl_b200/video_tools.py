"""Tensor-math helpers of the reference's file->file video paths, same names and signatures, on sm_90a kernels.

Reference: VRGDG_LUTVideoTools.py (_apply_lut_tensor :172-185, _apply_film_grain_tensor :262-277, uint8 codecs :736-752)
and VRGDG_StandaloneVideoEnhancerNodes.py (_auto_batch_size :200-210, _apply_unsharp :233-258, _apply_seeded_grain :261-275,
_apply_effects_batch :278-294).  The decode/encode, ffmpeg and HTTP route glue around them is out of scope.
"""
import ctypes

import numpy as np
import torch

from . import _native as nv
from . import ops
from ._runtime import compute_device, upload
from .chain import PostChain
from .lut_nodes import VRGDG_LUTS, _run_lut


def _to_cuda(t, device=None):
    dev = compute_device(t) if device in (None, "cpu", "auto") or str(device) == "cpu" else torch.device(device)
    return upload(t, dev), dev


def _apply_lut_tensor(image_tensor, lut_name, strength, device):
    """`device` is accepted for signature compatibility; compute is always CUDA, the result lands on the compute device
    like the reference's (which returns on `device`) unless that was "cpu" -> returned to the input's device."""
    lut_data = VRGDG_LUTS._load_lut(lut_name)
    src, dev = _to_cuda(image_tensor, device)
    out = _run_lut(src, lut_data, strength)
    return out if str(device) != "cpu" else out.to(image_tensor.device)


def _apply_film_grain_tensor(image_tensor, grain_intensity=0.04, saturation_mix=0.5, device="cpu", seed=None):
    intensity = max(0.0, min(1.0, float(grain_intensity)))
    saturation = max(0.0, min(1.0, float(saturation_mix)))
    src, dev = _to_cuda(image_tensor, device)
    if seed in (None, ""):
        seed = int(torch.randint(0, 2**62, (1,), dtype=torch.int64).item())
    out = ops.grain(src, intensity, saturation, 1.0 - saturation, int(seed), frame0=0, seed_mode=nv.SEED_PER_CLIP)
    return out if str(device) != "cpu" else out.to(image_tensor.device)


_ADJUST_FIELDS = {"temperature": (-100.0, 100.0), "tint": (-100.0, 100.0), "saturation": (-100.0, 100.0), "exposure": (-100.0, 100.0),
                  "contrast": (-100.0, 100.0), "highlights": (-100.0, 100.0), "shadows": (-100.0, 100.0), "whites": (-100.0, 100.0),
                  "blacks": (-100.0, 100.0), "sharpen": (0.0, 100.0), "clarity": (-100.0, 100.0), "vignette": (0.0, 100.0), "fade": (0.0, 100.0)}


def _normalize_adjust_settings(settings=None):
    """VRGDG_LUTVideoTools.py:280-304 (host logic): clamp every slider into its range, non-numeric -> 0."""
    settings = settings if isinstance(settings, dict) else {}
    out = {"enabled": settings.get("enabled", True) is not False}
    for key, (lo, hi) in _ADJUST_FIELDS.items():
        try:
            value = float(settings.get(key, 0.0))
        except Exception:
            value = 0.0
        out[key] = max(lo, min(hi, value))
    return out


def _adjust_desc(settings, height, width):
    """The scalars of _apply_adjust_tensor (:307-391), evaluated in double exactly as the reference's Python expressions do;
    ctypes rounds them to fp32 where torch rounds a Python scalar that meets an fp32 tensor."""
    a = _normalize_adjust_settings(settings)
    d = nv.AdjustDesc()
    d.enabled = 1 if a["enabled"] else 0
    d.offset_rgb = (ctypes.c_float * 3)(a["temperature"] / 400.0 - a["tint"] / 900.0, a["tint"] / 450.0, -a["temperature"] / 400.0 - a["tint"] / 900.0)
    d.exposure = 2.0 ** (a["exposure"] / 100.0)
    d.contrast = 1.0 + (a["contrast"] / 100.0)
    d.saturation = 1.0 + (a["saturation"] / 100.0)
    d.highlights, d.shadows = a["highlights"] / 220.0, a["shadows"] / 220.0
    d.whites, d.blacks = a["whites"] / 240.0, a["blacks"] / 240.0
    clarity, sharpen = a["clarity"] / 100.0, a["sharpen"] / 100.0
    d.clarity, d.sharpen = clarity, sharpen
    d.clarity_on = 1 if abs(clarity) > 0.001 else 0
    d.sharpen_on = 1 if sharpen > 0.001 else 0
    d.blur_kernel = min(9, height if height % 2 else height - 1, width if width % 2 else width - 1)
    if d.blur_kernel < 3:
        d.blur_kernel = 1                 # the reference's blur returns its input
    fade = a["fade"] / 100.0
    d.fade_on = 1 if fade > 0.0 else 0
    d.fade_mul, d.fade_add = 1.0 - fade * 0.35, fade * 0.18
    vignette = a["vignette"] / 100.0
    d.vignette_on = 1 if vignette > 0.0 else 0
    d.vignette = vignette
    return d


def _apply_adjust_tensor(image_tensor, settings=None, device="cpu"):
    """VRGDG_LUTVideoTools.py:307-391 on the GPU (bit-identical for fp32 frames); result on `device` like the reference, or on the
    input's device when that is "cpu"."""
    src, dev = _to_cuda(image_tensor, device)
    out = ops.adjust(src, _adjust_desc(settings, int(src.shape[1]), int(src.shape[2])))
    return out if str(device) != "cpu" else out.to(image_tensor.device)


def _auto_batch_size(width, height):
    """EnhancerNodes.py:200-210 (host logic, unchanged semantics)."""
    pixels = max(1, int(width) * int(height))
    for limit, batch in ((1280 * 720, 16), (1920 * 1080, 8), (2560 * 1440, 4), (3200 * 1800, 2)):
        if pixels <= limit:
            return batch
    return 1


def _resize_frames(frames, output_width, output_height):
    """EnhancerNodes.py:213-230: list of uint8 HWC frames -> list resized with cv2.INTER_LANCZOS4 semantics (bit-identical), frames
    already at the output size are passed through untouched.  One upload / two launches / one download per group of equal-sized
    frames; use ops.resize_lanczos4_u8 directly to stay on the device."""
    output_width, output_height = max(1, int(output_width)), max(1, int(output_height))
    resized = list(frames)
    todo = {}
    for i, frame in enumerate(frames):
        if not (frame.shape[1] == output_width and frame.shape[0] == output_height):
            todo.setdefault(tuple(frame.shape), []).append(i)
    dev = compute_device()
    for shape, idx in todo.items():
        if len(shape) != 3 or shape[2] != 3 or frames[idx[0]].dtype != np.uint8:
            raise ValueError("vrgdg_b200: _resize_frames expects uint8 [H,W,3] frames, got %s %s" % (shape, frames[idx[0]].dtype))
        batch = upload(torch.from_numpy(np.stack([np.ascontiguousarray(frames[i]) for i in idx])), dev)
        out = ops.resize_lanczos4_u8(batch, output_height, output_width).cpu().numpy()
        for j, i in enumerate(idx):
            resized[i] = out[j]
    return resized


def _apply_unsharp(images, strength, use_gpu):
    if strength <= 0:
        return images
    src, dev = _to_cuda(images)
    out = ops.stencil3x3(src, nv.STENCIL_BOX_UNSHARP, float(strength), nv.BORDER_ZERO if use_gpu else nv.BORDER_REPLICATE)
    return out.to(images.device)


def _apply_seeded_grain(images, intensity, saturation_mix, seed, frame_start):
    if intensity <= 0:
        return images
    src, dev = _to_cuda(images)
    s = float(saturation_mix)
    out = ops.grain(src, float(intensity), s, 1.0 - s, int(seed), frame0=int(frame_start), seed_mode=nv.SEED_PER_FRAME)
    return out.to(images.device)


def _apply_effects_batch(images, settings, frame_start=0):
    """unsharp (if enabled) then per-frame seeded grain (if enabled) in ONE fused kernel; returns a CPU tensor like
    the reference (:294)."""
    use_gpu = bool(settings.get("use_gpu", True))
    src, dev = _to_cuda(images)
    stencil = post = None
    if settings.get("sharpen_enabled", True) and float(settings.get("sharpen_strength", 0.5)) > 0:
        stencil = dict(op=nv.STENCIL_BOX_UNSHARP, strength=float(settings.get("sharpen_strength", 0.5)),
                       border=nv.BORDER_ZERO if use_gpu else nv.BORDER_REPLICATE)
    if settings.get("grain_enabled", False) and float(settings.get("grain_intensity", 0.04)) > 0:
        post = dict(intensity=float(settings.get("grain_intensity", 0.04)), saturation_mix=float(settings.get("saturation_mix", 0.5)),
                    seed=int(settings.get("seed", 42)), seed_mode=nv.SEED_PER_FRAME)
    if stencil is None and post is None:
        return images.detach().cpu()
    if stencil is None:
        s = post["saturation_mix"]
        out = ops.grain(src, post["intensity"], s, 1.0 - s, post["seed"], frame0=int(frame_start), seed_mode=nv.SEED_PER_FRAME)
    else:
        out = PostChain(stencil=stencil, post_grain=post, device=dev)(src, first_frame=int(frame_start))
    return out.detach().cpu()


def enhance_frames(frames, output_width, output_height, settings, frame_start=0):
    """The data path of one batch of the standalone enhancer's render loop (EnhancerNodes.py:415-420):
    `_tensor_to_frames(_apply_effects_batch(_frames_to_tensor(_resize_frames(frames, w, h)), settings, frame_start))`, bytes in ->
    bytes out, without leaving the GPU in between: one upload of the decoded uint8 BGR frames, Lanczos4 resize (2 launches, only if
    the size differs), unsharp + per-frame seeded grain directly on the bytes (1 launch), one download.  Byte-identical to the
    four helpers called one after the other."""
    output_width, output_height = max(1, int(output_width)), max(1, int(output_height))
    if not frames:
        return []
    shapes = {tuple(f.shape) for f in frames}
    if len(shapes) != 1 or len(next(iter(shapes))) != 3 or next(iter(shapes))[2] != 3 or any(f.dtype != np.uint8 for f in frames):
        # mixed sizes are legal for the reference (cv2 resizes frame by frame): take the helper-by-helper route
        return _tensor_to_frames(_apply_effects_batch(_frames_to_tensor(_resize_frames(frames, output_width, output_height)), settings, frame_start))
    dev = compute_device()
    batch = upload(torch.from_numpy(np.stack([np.ascontiguousarray(f) for f in frames], axis=0)), dev)
    if batch.shape[1] != output_height or batch.shape[2] != output_width:
        batch = ops.resize_lanczos4_u8(batch, output_height, output_width)
    use_gpu = bool(settings.get("use_gpu", True))
    stencil = post = None
    if settings.get("sharpen_enabled", True) and float(settings.get("sharpen_strength", 0.5)) > 0:
        stencil = dict(op=nv.STENCIL_BOX_UNSHARP, strength=float(settings.get("sharpen_strength", 0.5)),
                       border=nv.BORDER_ZERO if use_gpu else nv.BORDER_REPLICATE)
    if settings.get("grain_enabled", False) and float(settings.get("grain_intensity", 0.04)) > 0:
        post = dict(intensity=float(settings.get("grain_intensity", 0.04)), saturation_mix=float(settings.get("saturation_mix", 0.5)),
                    seed=int(settings.get("seed", 42)), seed_mode=nv.SEED_PER_FRAME)
    if stencil is not None:
        batch = PostChain(stencil=stencil, post_grain=post, device=dev)(batch, first_frame=int(frame_start))
    elif post is not None:
        s = post["saturation_mix"]
        batch = ops.grain(batch, post["intensity"], s, 1.0 - s, post["seed"], frame0=int(frame_start), seed_mode=nv.SEED_PER_FRAME)
    return list(batch.cpu().numpy())


def _frames_to_tensor(frames, device=None):
    """uint8 BGR frames (list of [H,W,3] arrays) -> float RGB [B,H,W,3] on the GPU: x/255 with the channel swap fused."""
    stacked = torch.from_numpy(np.stack(frames, axis=0))
    dev = compute_device() if device is None else torch.device(device)
    return ops.u8bgr_to_rgb(upload(stacked, dev))


def _tensor_to_frames(tensor):
    """float RGB -> list of uint8 BGR frames: clip(x*255, 0, 255) TRUNCATED (not rounded), as the reference does."""
    src, dev = _to_cuda(tensor.detach())
    return list(ops.rgb_to_u8bgr(src).cpu().numpy())

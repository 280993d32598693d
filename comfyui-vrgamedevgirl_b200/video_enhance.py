"""Resample helpers around the reference's Video Enhance nodes, same names and signatures, on one sm_90a gather kernel.

Reference: VRGDG_VideoEnhanceNodes.py (_interpolation :45-51, _resize_batch :54-86, _restore_batch :89-106, the restore blend of
VRGDG_VideoEnhanceRestore :404-418).  F.interpolate + crop / F.pad + clamp become ONE launch (vrgdg_resize): the fit mode only
changes the ROI, the resampled size and the placement offset handed to the kernel.  The LTX sampling between prepare and restore,
the context dict and the logging are the reference's control plane and stay out of scope.
"""

from . import ops
from ._runtime import compute_device, upload


def _interpolation(mode):
    return {"Nearest": "nearest", "Bilinear": "bilinear", "Bicubic (recommended)": "bicubic", "Area": "area"}.get(str(mode), "bicubic")


def _resize_plan(source_width, source_height, target_width, target_height, fit_mode):
    """(resampled (w, h), offset (x, y)) of _resize_batch's three fit modes (:66-85), Python arithmetic unchanged."""
    sw, sh, tw, th = int(source_width), int(source_height), int(target_width), int(target_height)
    if fit_mode == "Stretch to dimensions":
        return (tw, th), (0, 0)
    fill = fit_mode == "Crop to fill"
    scale = max(tw / sw, th / sh) if fill else min(tw / sw, th / sh)
    rw, rh = max(1, int(round(sw * scale))), max(1, int(round(sh * scale)))
    if fill:
        return (rw, rh), (-max(0, (rw - tw) // 2), -max(0, (rh - th) // 2))
    return (rw, rh), (max(0, (tw - rw) // 2), max(0, (th - rh) // 2))


def _output_size(resampled, offset, target_width, target_height, fit_mode):
    """Shape the reference's slicing / padding really produces (a crop never grows, a pad never shrinks)."""
    (rw, rh), (ox, oy) = resampled, offset
    if fit_mode == "Stretch to dimensions":
        return int(target_width), int(target_height)
    if fit_mode == "Crop to fill":
        return min(int(target_width), rw + ox), min(int(target_height), rh + oy)
    return max(int(target_width), rw), max(int(target_height), rh)


def _resize_batch(images, target_width, target_height, fit_mode, resize_method, _roi=None):
    if images.ndim != 4 or images.shape[0] < 1:
        raise ValueError("Video Enhance requires a non-empty IMAGE batch.")
    dev = compute_device(images)
    src = upload(images, dev)
    x0, y0, sw, sh = _roi if _roi is not None else (0, 0, int(src.shape[2]), int(src.shape[1]))
    resampled, offset = _resize_plan(sw, sh, target_width, target_height, fit_mode)
    ow, oh = _output_size(resampled, offset, target_width, target_height, fit_mode)
    out = ops.resize(src, oh, ow, _interpolation(resize_method), roi=(x0, y0, sw, sh), resampled=resampled, offset=offset)
    return out.to(images.device)


def _restore_batch(images, source_width, source_height, fit_mode, resize_method):
    if fit_mode != "Fit with letterbox (preserve all)":
        return _resize_batch(images, source_width, source_height, "Stretch to dimensions", resize_method)
    work_h, work_w = int(images.shape[1]), int(images.shape[2])
    scale = min(work_w / source_width, work_h / source_height)
    content_w = min(work_w, max(1, int(round(source_width * scale))))
    content_h = min(work_h, max(1, int(round(source_height * scale))))
    left, top = max(0, (work_w - content_w) // 2), max(0, (work_h - content_h) // 2)
    return _resize_batch(images, source_width, source_height, "Stretch to dimensions", resize_method,
                         _roi=(left, top, content_w, content_h))


def restore_frames(originals, enhanced, source_width, source_height, fit_mode, resize_method, enhancement_strength):
    """Tensor part of VRGDG_VideoEnhanceRestore.restore (:404-418): resample the enhanced frames back to the source size and lerp
    them over the originals; frames the sampler did not return keep the original (clamped)."""
    dev = compute_device(originals)
    orig = upload(originals, dev)
    restored = _restore_batch(upload(enhanced, dev), source_width, source_height, fit_mode, resize_method).to(orig.dtype)
    usable = min(int(orig.shape[0]), int(restored.shape[0]))
    strength = float(enhancement_strength)
    output = orig.clamp(0, 1)
    if usable > 0:
        output[:usable, ..., :3] = ops.blend(orig[:usable, ..., :3], restored[:usable], 1.0 - strength, strength)
    return output.to(originals.device)

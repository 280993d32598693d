"""Resample helpers around the reference's Video Enhance nodes, same names and signatures, on one sm_90a gather kernel.

Reference: VRGDG_VideoEnhanceNodes.py (_interpolation :45-51, _resize_batch :54-86, _restore_batch :89-106, the restore blend of
VRGDG_VideoEnhanceRestore :404-418).  F.interpolate + crop / F.pad + clamp become ONE launch (vrgdg_resize): the fit mode only
changes the ROI, the resampled size and the placement offset handed to the kernel; the restore's resample, blend and clamp are
one vrgdg_restore_blend launch per streamed chunk of originals.  The LTX sampling between prepare and restore,
the context dict and the logging are the reference's control plane and stay out of scope.
"""

from . import ops
from ._runtime import compute_device, devices_from_env, run_frames, upload


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
    """The result has the input's device and dtype.  A CUDA batch is one vrgdg_resize launch.  A host batch streams through
    run_frames like every frame node's IMAGE: VRGDG_STREAM_CHUNK_BYTES chunks (sized on the larger of an input and an output frame),
    sharded over VRGDG_DEVICES, one launch per chunk with the same plan, so device and pinned host memory follow the chunk, not the
    clip.  Every output frame depends only on its own input frame, so the result does not depend on the cut."""
    if images.ndim != 4 or images.shape[0] < 1:
        raise ValueError("Video Enhance requires a non-empty IMAGE batch.")
    dev = compute_device(images)
    x0, y0, sw, sh = _roi if _roi is not None else (0, 0, int(images.shape[2]), int(images.shape[1]))
    resampled, offset = _resize_plan(sw, sh, target_width, target_height, fit_mode)
    ow, oh = _output_size(resampled, offset, target_width, target_height, fit_mode)
    mode = _interpolation(resize_method)

    def make_fn(card):
        return lambda frames, first: ops.resize(frames, oh, ow, mode, roi=(x0, y0, sw, sh), resampled=resampled, offset=offset)

    devs = devices_from_env() if images.device.type == "cpu" else None
    return run_frames(images, make_fn, 0, images.device, dev, devs, out_frame_shape=(oh, ow, 3))


def _restore_roi(work_w, work_h, source_width, source_height, fit_mode):
    """(x0, y0, w, h) of the enhanced frame that _restore_batch resamples back to the source size (:89-106): the letterbox content,
    or the whole frame for the other fit modes."""
    if fit_mode != "Fit with letterbox (preserve all)":
        return 0, 0, int(work_w), int(work_h)
    scale = min(work_w / source_width, work_h / source_height)
    content_w = min(work_w, max(1, int(round(source_width * scale))))
    content_h = min(work_h, max(1, int(round(source_height * scale))))
    return max(0, (work_w - content_w) // 2), max(0, (work_h - content_h) // 2), content_w, content_h


def _restore_batch(images, source_width, source_height, fit_mode, resize_method):
    if fit_mode != "Fit with letterbox (preserve all)":
        return _resize_batch(images, source_width, source_height, "Stretch to dimensions", resize_method)
    roi = _restore_roi(int(images.shape[2]), int(images.shape[1]), source_width, source_height, fit_mode)
    return _resize_batch(images, source_width, source_height, "Stretch to dimensions", resize_method, _roi=roi)


def restore_frames(originals, enhanced, source_width, source_height, fit_mode, resize_method, enhancement_strength):
    """Tensor part of VRGDG_VideoEnhanceRestore.restore (:404-418): resample the enhanced frames back to the source size and lerp
    them over the originals; frames the sampler did not return keep the original (clamped).  The result has the originals' device,
    dtype and shape.

    The originals stream through run_frames like every other frame node's IMAGE (host batches in VRGDG_STREAM_CHUNK_BYTES chunks,
    sharded over VRGDG_DEVICES when the result is a host tensor too); each chunk uploads only the enhanced frames of the same
    absolute indices and makes one vrgdg_restore_blend launch, so device memory follows the chunk, not the clip.  Enhanced frames of
    another dtype than the originals take resize -> .to(dtype) -> blend per chunk: rounding the resample in the enhanced dtype
    first is part of that result."""
    if enhanced.ndim != 4 or enhanced.shape[0] < 1:
        raise ValueError("Video Enhance requires a non-empty IMAGE batch.")
    usable = min(int(originals.shape[0]), int(enhanced.shape[0]))
    H, W = int(source_height), int(source_width)
    if usable > 0 and (int(originals.shape[1]), int(originals.shape[2])) != (H, W):
        raise ValueError("Video Enhance: the context's source size %dx%d differs from the original frames' %dx%d"
                         % (W, H, int(originals.shape[2]), int(originals.shape[1])))
    roi = _restore_roi(int(enhanced.shape[2]), int(enhanced.shape[1]), source_width, source_height, fit_mode)
    mode = _interpolation(resize_method)
    strength = float(enhancement_strength)
    fused = enhanced.dtype == originals.dtype and int(originals.shape[-1]) in (3, 4)

    def make_fn(card):
        def fn(orig, first):
            n = max(0, min(first + int(orig.shape[0]), usable) - first)
            enh = upload(enhanced[first:first + n], card)              # the same absolute frames; empty past the last one
            if fused:
                return ops.restore_blend(enh, orig, mode, 1.0 - strength, strength, roi=roi, n_restored=n)
            out = orig.clamp(0, 1)
            if n > 0:
                restored = ops.resize(enh, H, W, mode, roi=roi).to(orig.dtype)
                out[:n, ..., :3] = ops.blend(orig[:n, ..., :3], restored, 1.0 - strength, strength)
            return out
        return fn

    dev = compute_device(originals)
    devs = devices_from_env() if originals.device.type == "cpu" else None
    return run_frames(originals, make_fn, 0, originals.device, dev, devs)

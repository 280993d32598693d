"""Graph-reachable entries to the fused kernels and the video-enhance tensor paths.

* VRGDGVideoEnhanceRestoreOriginal, VRGDGStandaloneVideoEnhancer: the REFERENCE's node keys, INPUT_TYPES, RETURN_* and method
  signatures (VRGDG_VideoEnhanceNodes.py:378-437, VRGDG_StandaloneVideoEnhancerNodes.py:869-903), so saved workflows load unchanged.
* VRGDG_B200_PostChain, VRGDG_B200_EnhanceFrames, VRGDG_B200_TemporalSharpen, VRGDG_B200_HistogramColorMatch: EXTRA keys (nothing in the reference has them).  A workflow that chains
  FastFilmGrain -> ColorMatchToReference -> VRGDG_LUTS -> FastUnsharpSharpen as four nodes pays four launches and, with ComfyUI's
  CPU intermediate device, four PCIe round trips; VRGDG_B200_PostChain is the same arithmetic (same widgets, same order) as ONE
  upload, the fused kernels, one download.  bench.py reports both (`e2e` and `e2e.stock_nodes`).
"""
import torch

from . import _native as nv
from ._runtime import compute_device, devices_from_env, grain_noise_from_env, result_device, run_frames, upload
from .chain import PostChain
from .filter_nodes import GlobalStreamDraws, _as_frames, draw_seed
from .lut_nodes import NO_LUTS, VRGDG_LUTS, _list_lut_files
from .video_enhance import restore_frames

VIDEO_ENHANCE_CONTEXT = "VRGDG_VIDEO_ENHANCE_CONTEXT"      # VRGDG_VideoEnhanceNodes.py:12
_NONE = "none"
_SHARPENERS = {
    _NONE: (nv.STENCIL_NONE, nv.STENCIL_NONE),
    "unsharp": (nv.STENCIL_BOX_UNSHARP, nv.STENCIL_BOX_UNSHARP),
    "laplacian": (nv.STENCIL_LAPLACIAN_CPU, nv.STENCIL_LAPLACIAN_GPU),
    "sobel": (nv.STENCIL_SOBEL_CPU, nv.STENCIL_SOBEL_GPU),
}


class VRGDG_B200_PostChain:
    """grain -> [colour match] -> 3D LUT -> sharpen in one pass over HBM (chain.PostChain).  Stage semantics and widget ranges
    are those of the four reference nodes (nodes.py:20-34, :72-84, :135-147; VRGDG_IV_Adjustments.py:145-157).  RGBA batches take
    the LUT and the sharpeners the reference runs on 4 channels: grain_intensity 0, no reference_image, and use_gpu=False for
    laplacian / sobel.  reference_image holds one frame or one per frame, as ColorMatchToReference's does: with B frames, frame i is
    matched to reference frame i at every batch_size, and each chunk uploads only its own reference frames.  With VRGDG_GRAIN_NOISE=torch_cuda (read at call time) the grain is FastFilmGrain(images, grain_intensity,
    saturation_mix, batch_size)'s in that mode, drawn from the compute device's global CUDA generator, which is advanced as that
    node advances it."""

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "images": ("IMAGE",),
                "grain_intensity": ("FLOAT", {"default": 0.04, "min": 0.0, "max": 1.0, "step": 0.001, "tooltip": "0 disables the grain stage"}),
                "saturation_mix": ("FLOAT", {"default": 0.5, "min": 0.0, "max": 1.0, "step": 0.01}),
                "match_strength": ("FLOAT", {"default": 1.0, "min": 0.0, "max": 1.0, "step": 0.01, "tooltip": "used only when reference_image is connected"}),
                "lut_name": ([_NONE] + [n for n in _list_lut_files() if n != NO_LUTS],),
                "lut_strength": ("FLOAT", {"default": 10.0, "min": 0.0, "max": 10.0, "step": 0.1}),
                "sharpen": (list(_SHARPENERS), {"default": "unsharp"}),
                "sharpen_strength": ("FLOAT", {"default": 0.5, "min": 0.0, "max": 10.0, "step": 0.01}),
                "use_gpu": ("BOOLEAN", {"default": False, "tooltip": "False: the reference's NumPy-path semantics (edge-replicated border); True: its torch path (zero padding)"}),
                "batch_size": ("INT", {"default": 8, "min": 0, "max": 500, "step": 1, "tooltip": "frames per upload chunk (device memory bound); results do not depend on it, except with VRGDG_GRAIN_NOISE=torch_cuda, where it is also the grain's draw size (0 = the whole batch), as FastFilmGrain's batch_size is"}),
            },
            "optional": {"reference_image": ("IMAGE",)},
        }

    RETURN_TYPES = ("IMAGE",)
    FUNCTION = "apply_chain"
    CATEGORY = "video/enhancement"
    DESCRIPTION = "Film grain, colour match, 3D LUT and sharpen fused into one GPU pass (H100)."

    def apply_chain(self, images, grain_intensity, saturation_mix, match_strength, lut_name, lut_strength, sharpen, sharpen_strength, use_gpu,
                    batch_size, reference_image=None):
        images = _as_frames(images, channels=(3, 4))
        if images.shape[-1] == 4:
            # RGBA: the stages the reference runs on 4 channels, VRGDG_LUTS and the NumPy-path sharpeners (the grain's gray
            # broadcast, kornia's colour conversion and the torch-path conv2d with groups=3 raise there)
            if float(grain_intensity) > 0:
                raise ValueError("VRGDG_B200_PostChain: grain_intensity must be 0 for RGBA images (film grain takes 3 channels), got 4 channels")
            if reference_image is not None:
                raise ValueError("VRGDG_B200_PostChain: reference_image (colour match) takes 3-channel images, got 4 channels; disconnect it")
            if use_gpu and _SHARPENERS[sharpen][1] in (nv.STENCIL_LAPLACIAN_GPU, nv.STENCIL_SOBEL_GPU):
                raise ValueError("VRGDG_B200_PostChain: sharpen=%s with use_gpu=True takes 3-channel images (the torch path convolves "
                                 "with groups=3), got 4 channels" % sharpen)
        ref = n_ref = None
        if reference_image is not None:
            # ColorMatchToReference's rule: one reference frame for every frame, or one per frame (frame i matched to reference i)
            ref = _as_frames(reference_image, "reference_image")
            n_ref = int(ref.shape[0])
            if n_ref != 1 and n_ref != int(images.shape[0]):
                raise ValueError("reference_image batch (%d) must be 1 or match images batch (%d)" % (n_ref, images.shape[0]))
        # the global stream's refusals come before any generator or device work
        draws = GlobalStreamDraws(images, batch_size, "VRGDG_B200_PostChain") \
            if float(grain_intensity) > 0 and grain_noise_from_env() == "torch_cuda" else None
        dev = compute_device(images)
        grain = None
        if draws is None and float(grain_intensity) > 0:
            grain = dict(intensity=float(grain_intensity), saturation_mix=float(saturation_mix), seed=draw_seed())
        cm = None
        if reference_image is not None:
            if n_ref == 1:
                cm = dict(reference_image=ref.to(images.dtype), strength=float(match_strength))
            else:       # streamed: each chunk uploads the reference frames of its own indices
                cm = dict(reference_frames=ref, strength=float(match_strength))
        lut = None
        if lut_name != _NONE and float(lut_strength) > 0:
            lut = dict(lut_data=VRGDG_LUTS._load_lut(lut_name), strength=float(lut_strength))
        stencil = None
        op = _SHARPENERS[sharpen][1 if use_gpu else 0]
        if op != nv.STENCIL_NONE:
            stencil = dict(op=op, strength=float(sharpen_strength), border=nv.BORDER_ZERO if use_gpu else nv.BORDER_REPLICATE)
        if grain is None and draws is None and cm is None and lut is None and stencil is None:
            return (images,)
        devs = devices_from_env() if images.device.type == "cpu" else None
        if draws is not None:
            grain = dict(intensity=float(grain_intensity), saturation_mix=float(saturation_mix), torch_global=draws.snapshot(images)[1])
        chain = PostChain(grain=grain, colormatch=cm, lut=lut, stencil=stencil, device=None if devs else dev, devices=devs)
        out = run_frames(images, chain.make_fn(), batch_size, result_device(images), chain.device, devs)
        if draws is not None:
            draws.advance()
        return (out,)


class VRGDG_B200_EnhanceFrames:
    """Tensor form of the standalone enhancer's per-batch data path (_apply_effects_batch, EnhancerNodes.py:278-294): unsharp, then
    per-frame seeded grain, one fused kernel."""

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "images": ("IMAGE",),
                "sharpen_strength": ("FLOAT", {"default": 0.5, "min": 0.0, "max": 10.0, "step": 0.01}),
                "grain_intensity": ("FLOAT", {"default": 0.04, "min": 0.0, "max": 1.0, "step": 0.001}),
                "saturation_mix": ("FLOAT", {"default": 0.5, "min": 0.0, "max": 1.0, "step": 0.01}),
                "seed": ("INT", {"default": 42, "min": 0, "max": 0x7FFFFFFF}),
                "frame_start": ("INT", {"default": 0, "min": 0, "max": 0x7FFFFFFF}),
                "use_gpu": ("BOOLEAN", {"default": True, "tooltip": "the enhancer's setting of the same name: True = zero-padded box blur (avg_pool2d), False = edge-replicated"}),
            },
            "optional": {
                "noise_stream": (["vrgdg", "torch_cuda"], {"default": "vrgdg", "tooltip": "vrgdg = this package's grain generator; torch_cuda = "
                                 "torch's CUDA randn stream of the enhancer's per-frame seeded generators: the same grain as the reference "
                                 "rendering on the same GPU model"}),
            },
        }

    RETURN_TYPES = ("IMAGE",)
    FUNCTION = "enhance"
    CATEGORY = "VRGDG/Video"
    DESCRIPTION = "Unsharp + per-frame seeded film grain (the standalone enhancer's effect chain) on an IMAGE batch."

    def enhance(self, images, sharpen_strength, grain_intensity, saturation_mix, seed, frame_start, use_gpu, noise_stream="vrgdg"):
        from .video_tools import _seed_mode
        mode = _seed_mode(noise_stream, nv.SEED_PER_FRAME, nv.SEED_TORCH_PER_FRAME)
        images = _as_frames(images)
        dev = compute_device(images)
        stencil = dict(op=nv.STENCIL_BOX_UNSHARP, strength=float(sharpen_strength), border=nv.BORDER_ZERO if use_gpu else nv.BORDER_REPLICATE) \
            if float(sharpen_strength) > 0 else None
        post = dict(intensity=float(grain_intensity), saturation_mix=float(saturation_mix), seed=int(seed), seed_mode=mode) \
            if float(grain_intensity) > 0 else None
        if stencil is None and post is None:
            return (images,)
        devs = devices_from_env() if images.device.type == "cpu" else None
        if stencil is None:
            from . import ops
            s = post["saturation_mix"]
            make_fn = lambda d: lambda f, i: ops.grain(f, post["intensity"], s, 1.0 - s, post["seed"], frame0=int(frame_start) + i,
                                                       seed_mode=mode)
        else:
            make_fn = PostChain(stencil=stencil, post_grain=post, device=None if devs else dev, devices=devs).make_fn(int(frame_start))
        return (run_frames(images, make_fn, 8, result_device(images), devs[0] if devs else dev, devs),)


class VRGDG_B200_HistogramColorMatch:
    """Histogram / CDF colour transfer to a reference image: per-channel 256-bin histograms, monotone CDF mapping (the colour-match
    mode BASELINE.json describes).  An extension of this package: the reference's ColorMatchToReference is the LAB mean/std transfer
    and stays that; the arithmetic of this mode is specified in include/vrgdg_b200.h (vrgdg_hist_counts ...).  reference_image holds
    one frame or one per frame, as ColorMatchToReference's does: with B frames, frame i is matched to reference frame i at every
    batch_size, and each chunk uploads only its own reference frames (vrgdg_histmatch_apply_refs), so the clip never has to fit
    on the card."""

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "images": ("IMAGE",),
                "reference_image": ("IMAGE",),
                "match_strength": ("FLOAT", {"default": 1.0, "min": 0.0, "max": 1.0, "step": 0.01}),
                "batch_size": ("INT", {"default": 8, "min": 0, "max": 500, "step": 1}),
            }
        }

    RETURN_TYPES = ("IMAGE",)
    FUNCTION = "match_histogram"
    CATEGORY = "video/enhancement"
    DESCRIPTION = "Matches each frame's per-channel histogram to a reference image (monotone CDF transfer, H100)."

    def match_histogram(self, images, reference_image, match_strength, batch_size):
        from . import ops
        images = _as_frames(images)
        ref = _as_frames(reference_image, "reference_image")
        n_ref = int(ref.shape[0])
        if n_ref != 1 and n_ref != int(images.shape[0]):
            raise ValueError("reference_image batch (%d) must be 1 or match images batch (%d)" % (n_ref, images.shape[0]))
        dev = compute_device(images)
        t = float(match_strength)
        ref_counts = None
        if n_ref == 1:
            with torch.cuda.device(dev):
                ref_counts = ops.hist_counts(upload(ref, dev).to(images.dtype))

        def make_fn(card):
            if n_ref == 1:
                counts = ref_counts.to(card)         # made once, copied to each card
                def run(frames, first):
                    tables = ops.histmatch_tables(ops.hist_counts(frames), counts)
                    return ops.histmatch_apply(frames, tables, t, 1.0 - t)
                return run
            # a reference clip stays where the caller keeps it; each chunk uploads the reference frames of its own absolute indices
            # and converts them on its card.  The scratch is the worker's own (two workers on one card must not share one)
            state = {"scratch": None}
            def run_clip(frames, first):
                refs = upload(ref[first:first + frames.shape[0]], card).to(frames.dtype)
                out, state["scratch"] = ops.histmatch_apply_refs(frames, refs, t, 1.0 - t, scratch=state["scratch"])
                return out
            return run_clip
        devs = devices_from_env() if images.device.type == "cpu" else None
        return (run_frames(images, make_fn, batch_size, result_device(images), dev, devs),)


class VRGDG_B200_TemporalSharpen:
    """3-frame temporal unsharp over an IMAGE batch read as a clip (BASELINE.json configs[4]).  An extension of this package: the
    reference has no temporal operator, the arithmetic is specified in include/vrgdg_b200.h (vrgdg_temporal_sharpen)."""

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "images": ("IMAGE",),
                "strength": ("FLOAT", {"default": 0.5, "min": 0.0, "max": 10.0, "step": 0.01}),
                "batch_size": ("INT", {"default": 16, "min": 0, "max": 500, "step": 1, "tooltip": "frames per upload chunk; chunks carry their neighbour frames, results do not depend on it"}),
            }
        }

    RETURN_TYPES = ("IMAGE",)
    FUNCTION = "sharpen"
    CATEGORY = "video/enhancement"
    DESCRIPTION = "Temporal unsharp mask: each frame is sharpened against the mean of itself and its two neighbours (H100)."

    def sharpen(self, images, strength, batch_size):
        from . import ops
        images = _as_frames(images)
        dev = compute_device(images)
        T = int(images.shape[0])
        if T == 0 or float(strength) == 0.0:
            return (images,)
        s = float(strength)

        def make_fn(card):
            def run(frames, first):      # the chunk's neighbours come from the clip itself (host or device tensor), by absolute index
                n = int(frames.shape[0])
                prev = images[first - 1].to(card) if first > 0 else None
                nxt = images[first + n].to(card) if first + n < T else None
                return ops.temporal_sharpen(frames, s, prev, nxt)
            return run
        devs = devices_from_env() if images.device.type == "cpu" else None
        return (run_frames(images, make_fn, batch_size, result_device(images), dev, devs),)


class VRGDGVideoEnhanceRestoreOriginal:
    """VRGDG_VideoEnhanceNodes.py:378-419: resample the LTX output back to the source size and blend it over the originals."""

    @classmethod
    def INPUT_TYPES(cls):
        return {"required": {
            "ltx_enhanced_frames": ("IMAGE", {"tooltip": "Connect the final decoded IMAGE batch from LTX. These temporary working-resolution frames are resized back to the exact source dimensions."}),
            "video_enhance_context": (VIDEO_ENHANCE_CONTEXT, {"tooltip": "Connect Collect LTX Inputs context. It contains the untouched source frames, exact source dimensions, and frame count."}),
            "resize_method": (["Bicubic (recommended)", "Bilinear", "Area", "Nearest"], {"default": "Bicubic (recommended)", "tooltip": "Interpolation used to restore LTX frames to the exact source width and height. This changes dimensions only; optional AI upscalers may be inserted before this node if desired."}),
            "enhancement_strength": ("FLOAT", {"default": 1.0, "min": 0.0, "max": 1.0, "step": 0.05, "tooltip": "Blends the restored LTX result with the untouched original video. 1 uses the complete LTX result; lower values retain more original pixels and can reduce over-processing."}),
        }}

    RETURN_TYPES = ("IMAGE", "INT", "INT", "INT", "FLOAT")
    RETURN_NAMES = ("enhanced_video_frames", "frame_count", "original_width", "original_height", "fps")
    FUNCTION = "restore"
    CATEGORY = "VRGameDevGirl/Video Enhance"
    DESCRIPTION = "Restores decoded LTX output to the exact input resolution and frame count, preserving unmatched source-tail frames and optionally blending with the untouched source video."

    def restore(self, ltx_enhanced_frames, video_enhance_context, resize_method, enhancement_strength):
        originals = video_enhance_context.get("original_frames")
        if not isinstance(originals, torch.Tensor) or originals.ndim != 4:
            raise ValueError("Video Enhance context does not contain valid original frames.")
        source_height = int(video_enhance_context.get("source_height") or originals.shape[1])
        source_width = int(video_enhance_context.get("source_width") or originals.shape[2])
        frame_count = int(video_enhance_context.get("frame_count") or originals.shape[0])
        delta = frame_count - int(ltx_enhanced_frames.shape[0])
        if abs(delta) > 7:
            raise ValueError(f"LTX returned {ltx_enhanced_frames.shape[0]} frames for {frame_count} source frames.")
        fit_mode = str(video_enhance_context.get("fit_mode") or "Stretch to dimensions")
        output = restore_frames(originals, ltx_enhanced_frames[:frame_count], source_width, source_height, fit_mode, resize_method,
                                float(enhancement_strength))
        return output, frame_count, source_width, source_height, float(video_enhance_context.get("fps") or 0.0)


class VRGDGStandaloneVideoEnhancer:
    """VRGDG_StandaloneVideoEnhancerNodes.py:869-894: the graph node only hands the UI's output path on (the render itself is the
    route-driven job whose per-batch data path is video_tools.enhance_frames)."""

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "output_path": (
                    "STRING",
                    {
                        "default": "",
                        "multiline": False,
                        "tooltip": "Updated by the standalone UI after a successful render.",
                    },
                ),
            }
        }

    RETURN_TYPES = ("STRING",)
    RETURN_NAMES = ("enhanced_video_path",)
    FUNCTION = "return_output"
    OUTPUT_NODE = True
    CATEGORY = "VRGDG/Video"
    DESCRIPTION = "Standalone batched 2K–4K resize, video sharpening, film grain, and before/after comparison UI."

    def return_output(self, output_path):
        return (str(output_path or ""),)


NODE_CLASS_MAPPINGS = {
    "VRGDGVideoEnhanceRestoreOriginal": VRGDGVideoEnhanceRestoreOriginal,
    "VRGDGStandaloneVideoEnhancer": VRGDGStandaloneVideoEnhancer,
    "VRGDG_B200_PostChain": VRGDG_B200_PostChain,
    "VRGDG_B200_EnhanceFrames": VRGDG_B200_EnhanceFrames,
    "VRGDG_B200_TemporalSharpen": VRGDG_B200_TemporalSharpen,
    "VRGDG_B200_HistogramColorMatch": VRGDG_B200_HistogramColorMatch,
}
NODE_DISPLAY_NAME_MAPPINGS = {
    "VRGDGVideoEnhanceRestoreOriginal": "Video Enhance - Restore Original Resolution",
    "VRGDGStandaloneVideoEnhancer": "VRGDG Standalone Video Enhancer",
    "VRGDG_B200_PostChain": "VRGDG B200 Post Chain (grain + colour match + LUT + sharpen, fused)",
    "VRGDG_B200_EnhanceFrames": "VRGDG B200 Enhance Frames (unsharp + seeded grain, fused)",
    "VRGDG_B200_TemporalSharpen": "VRGDG B200 Temporal Sharpen (3-frame)",
    "VRGDG_B200_HistogramColorMatch": "VRGDG B200 Histogram Color Match (CDF transfer)",
}

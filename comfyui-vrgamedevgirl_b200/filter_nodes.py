"""The five per-pixel filter nodes of the reference's nodes.py (:18-384) on sm_90a kernels.

Node keys, INPUT_TYPES (widget order, defaults, ranges), RETURN_TYPES, FUNCTION names, CATEGORY and method
signatures are the reference's, so saved workflows load unchanged.  The arithmetic runs in libvrgdg_b200.so;
there is no CPU implementation in this package.
"""
from typing import Tuple

import torch

from . import _native as nv
from . import ops
from ._runtime import compute_device, result_device, stream_frames, upload

_FLOATS = (torch.float32, torch.float16, torch.bfloat16)


def _as_frames(images, name="images"):
    if not isinstance(images, torch.Tensor) or images.ndim != 4 or images.shape[-1] != 3:
        raise ValueError("%s must be an IMAGE tensor shaped [batch, height, width, 3]" % name)
    if images.dtype not in _FLOATS:
        images = images.float()
    return images


def draw_seed():
    """One 63-bit seed from torch's global CPU generator, so torch.manual_seed() makes FastFilmGrain
    reproducible the way it makes the reference's torch.randn_like (nodes.py:51) reproducible."""
    return int(torch.randint(0, 2**62, (1,), dtype=torch.int64).item())


class FastFilmGrain:
    """nodes.py:18-66."""

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "images": ("IMAGE",),
                "grain_intensity": ("FLOAT", {"default": 0.04, "min": 0.001, "max": 1.0, "step": 0.001}),
                "saturation_mix": ("FLOAT", {"default": 0.5, "min": 0.0, "max": 1.0, "step": 0.01}),
                "batch_size": ("INT", {"default": 4, "min": 0, "max": 500, "step": 1}),
            }
        }

    RETURN_TYPES = ("IMAGE",)
    FUNCTION = "apply_grain"
    CATEGORY = "video/enhancement"
    DESCRIPTION = "Adds lightweight film grain"

    def apply_grain(self, images, grain_intensity, saturation_mix, batch_size):
        images = _as_frames(images)
        seed = draw_seed()
        sat = float(saturation_mix)
        # batch_size only bounds device memory while streaming host frames; the noise is keyed by the absolute
        # frame index, so the result does not depend on it (0 = whole batch, nodes.py:46)
        def run(frames, first):
            return ops.grain(frames, grain_intensity, sat, 1.0 - sat, seed, frame0=first, seed_mode=nv.SEED_PER_CLIP)
        out = stream_frames(images, run, batch_size, result_device(images), compute_device(images))
        return (out,)


class ColorMatchToReference:
    """nodes.py:70-124: Reinhard LAB mean/std transfer to one reference image."""

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "images": ("IMAGE",),
                "reference_image": ("IMAGE",),
                "match_strength": ("FLOAT", {"default": 1.0, "min": 0.0, "max": 1.0, "step": 0.01}),
                "batch_size": ("INT", {"default": 1, "min": 1, "max": 500, "step": 1}),
            }
        }

    RETURN_TYPES = ("IMAGE",)
    FUNCTION = "match_color"
    CATEGORY = "video/enhancement"
    DESCRIPTION = "Matches the color tone of input image to a reference image using LAB mean/std alignment"

    def match_color(self, images, reference_image, match_strength, batch_size):
        images = _as_frames(images)
        reference_image = _as_frames(reference_image, "reference_image")
        n_ref = int(reference_image.shape[0])
        if n_ref != 1 and n_ref != int(images.shape[0]):
            raise ValueError("reference_image batch (%d) must be 1 or match images batch (%d)" % (n_ref, images.shape[0]))
        dev = compute_device(images)
        t = float(match_strength)
        with torch.cuda.device(dev):
            ref_sums = ops.lab_moments(upload(reference_image, dev).to(images.dtype))
        d = nv.ChainDesc()
        d.colormatch_enabled, d.cm_t, d.cm_one_minus_t = 1, t, 1.0 - t
        state = {"scratch": None}
        def run(frames, first):
            # one library call per chunk: statistics, parameters and the apply pass (which starts from the stored Lab f-planes for
            # fp32 frames instead of repeating the forward transform)
            rs = ref_sums if n_ref == 1 else ref_sums[first:first + frames.shape[0]]
            out, state["scratch"] = ops.chain_cm_apply(frames, d, rs, scratch=state["scratch"])
            return out
        out = stream_frames(images, run, batch_size, result_device(images), dev)
        return (out,)


class _StencilNode:
    OP_CPU = nv.STENCIL_NONE
    OP_GPU = nv.STENCIL_NONE

    def _apply(self, images, strength, use_gpu):
        images = _as_frames(images)
        # use_gpu=False -> the numpy path's semantics (edge-replicated border); True -> the torch path's (zero padding).
        op = self.OP_GPU if use_gpu else self.OP_CPU
        border = nv.BORDER_ZERO if use_gpu else nv.BORDER_REPLICATE
        s = float(strength)
        def run(frames, first):
            return ops.stencil3x3(frames, op, s, border)
        out = stream_frames(images, run, 8, result_device(images, numpy_path=not use_gpu), compute_device(images))
        return (out,)


class FastUnsharpSharpen(_StencilNode):
    """nodes.py:129-209: 3x3 box unsharp mask."""

    OP_CPU = nv.STENCIL_BOX_UNSHARP
    OP_GPU = nv.STENCIL_BOX_UNSHARP

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "images": ("IMAGE",),
                "strength": ("FLOAT", {"default": 0.5, "min": 0.0, "max": 10.0, "step": 0.01}),
                "use_gpu": ("BOOLEAN", {"default": False}),
            }
        }

    RETURN_TYPES = ("IMAGE",)
    FUNCTION = "apply_unsharp"
    CATEGORY = "video/enhancement"
    DESCRIPTION = "Unsharp mask (CPU default, optional GPU path)."

    def apply_unsharp(self, images: torch.Tensor, strength: float, use_gpu: bool) -> Tuple[torch.Tensor]:
        return self._apply(images, strength, use_gpu)


class FastLaplacianSharpen(_StencilNode):
    """nodes.py:212-289.  The two reference paths differ in sign (SURVEY D5); both are reproduced."""

    OP_CPU = nv.STENCIL_LAPLACIAN_CPU
    OP_GPU = nv.STENCIL_LAPLACIAN_GPU

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "images": ("IMAGE",),
                "strength": ("FLOAT", {"default": 0.5, "min": 0.0, "max": 2.0, "step": 0.01}),
                "use_gpu": ("BOOLEAN", {"default": False}),
            }
        }

    RETURN_TYPES = ("IMAGE",)
    FUNCTION = "apply_laplacian"
    CATEGORY = "video/enhancement"
    DESCRIPTION = "Laplacian sharpen (CPU default, optional GPU)."

    def apply_laplacian(self, images: torch.Tensor, strength: float, use_gpu: bool) -> Tuple[torch.Tensor]:
        return self._apply(images, strength, use_gpu)


class FastSobelSharpen(_StencilNode):
    """nodes.py:292-384."""

    OP_CPU = nv.STENCIL_SOBEL_CPU
    OP_GPU = nv.STENCIL_SOBEL_GPU

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "images": ("IMAGE",),
                "strength": ("FLOAT", {"default": 0.5, "min": 0.0, "max": 2.0, "step": 0.01}),
                "use_gpu": ("BOOLEAN", {"default": False}),
            }
        }

    RETURN_TYPES = ("IMAGE",)
    FUNCTION = "apply_sobel"
    CATEGORY = "video/enhancement"
    DESCRIPTION = "Sobel sharpen (CPU default, optional GPU)."

    def apply_sobel(self, images: torch.Tensor, strength: float, use_gpu: bool) -> Tuple[torch.Tensor]:
        return self._apply(images, strength, use_gpu)

"""The five per-pixel filter nodes of the reference's nodes.py (:18-384) on sm_90a kernels.

Node keys, INPUT_TYPES (widget order, defaults, ranges), RETURN_TYPES, FUNCTION names, CATEGORY and method
signatures are the reference's, so saved workflows load unchanged.  The arithmetic runs in libvrgdg_b200.so;
there is no CPU implementation in this package.
"""
from typing import Tuple

import torch

from . import _native as nv
from . import ops
from ._runtime import compute_device, cuda_device, devices_from_env, grain_noise_from_env, result_device, run_frames, upload

_FLOATS = (torch.float32, torch.float16, torch.bfloat16)


def _as_frames(images, name="images", channels=(3,)):
    if not isinstance(images, torch.Tensor) or images.ndim != 4 or images.shape[-1] not in channels:
        raise ValueError("%s must be an IMAGE tensor shaped [batch, height, width, %s]" % (name, " or ".join(map(str, channels))))
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
        if grain_noise_from_env() == "torch_cuda":
            return (_global_stream_grain(images, grain_intensity, float(saturation_mix), batch_size),)
        seed = draw_seed()
        sat = float(saturation_mix)
        # batch_size only bounds device memory while streaming host frames; the noise is keyed by the absolute
        # frame index, so the result does not depend on it (0 = whole batch, nodes.py:46)
        def run(frames, first):
            return ops.grain(frames, grain_intensity, sat, 1.0 - sat, seed, frame0=first, seed_mode=nv.SEED_PER_CLIP)
        devs = devices_from_env() if images.device.type == "cpu" else None
        out = run_frames(images, lambda dev: run, batch_size, result_device(images), compute_device(images), devs)
        return (out,)


class GlobalStreamDraws:
    """The generator bookkeeping of grain drawn as FastFilmGrain draws it under VRGDG_GRAIN_NOISE=torch_cuda (nodes.py:46-62 on a CUDA
    device): torch.randn_like once per mini-batch of batch_size frames (0 = the whole batch) from the compute device's global CUDA
    generator, which those draws leave advanced.  The constructor only checks the draws (a draw past 32-bit indexing raises
    ValueError) and touches neither a generator nor a device; snapshot() reads the generator, advance() moves it past the draws
    afterwards.  The CPU generator is never touched (the reference does not touch it either)."""

    def __init__(self, images, batch_size, who):
        B, H, W = (int(s) for s in images.shape[:3])
        self.B, self.n = B, H * W * 3
        self.step = min(int(batch_size), B) if int(batch_size) > 0 else B      # nodes.py:46; one draw when batch_size >= B
        if B > 0 and self.n > 0 and 1 + (self.step * self.n - 1) * images.element_size() > 2**31 - 1:
            raise ValueError("vrgdg_b200: %s with VRGDG_GRAIN_NOISE=torch_cuda: a draw of %d frames of %dx%d (batch_size=%d) exceeds "
                             "32-bit indexing (torch splits such a draw into sub-draws, which is not reproduced); lower batch_size"
                             % (who, self.step, W, H, int(batch_size)))
        self._gen = None

    def snapshot(self, images):
        """(device, dict(seed, philox_offset, clip_frames, draw_frames)): the compute device's generator as the draws find it"""
        dev = cuda_device(compute_device(images))
        torch.cuda.init()
        self._gen = torch.cuda.default_generators[dev.index]
        self._offset = self._gen.get_offset()
        self._total = 0
        if self.B > 0 and self.n > 0:
            self._total = (self.B // self.step) * ops.torch_randn_increment(self.step * self.n, dev) + \
                ops.torch_randn_increment((self.B % self.step) * self.n, dev)
        return dev, dict(seed=self._gen.initial_seed(), philox_offset=self._offset, clip_frames=self.B, draw_frames=self.step)

    def advance(self):
        """the generator's offset after the draws, as the reference's draws leave it"""
        self._gen.set_offset(self._offset + self._total)


def _global_stream_grain(images, intensity, sat, batch_size):
    """FastFilmGrain with VRGDG_GRAIN_NOISE=torch_cuda: the noise the reference draws on a CUDA device (GlobalStreamDraws).  Unlike
    the default path, the grain here depends on batch_size, as the reference's does."""
    draws = GlobalStreamDraws(images, batch_size, "FastFilmGrain")
    dev, g = draws.snapshot(images)

    def run(frames, first):
        return ops.grain_torch_global(frames, intensity, sat, 1.0 - sat, g["seed"], g["philox_offset"], first, g["clip_frames"], g["draw_frames"])
    devs = devices_from_env() if images.device.type == "cpu" else None
    out = run_frames(images, lambda card: run, batch_size, result_device(images), dev, devs)
    draws.advance()
    return out


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
        ref_sums = None
        if n_ref == 1:
            with torch.cuda.device(dev):
                ref_sums = ops.lab_moments(upload(reference_image, dev).to(images.dtype))
        d = nv.ChainDesc()
        d.colormatch_enabled, d.cm_t, d.cm_one_minus_t = 1, t, 1.0 - t

        def make_fn(card):
            # one reference: its sums are made once and copied to each card.  A reference clip (n_ref == B) stays where the caller
            # keeps it; each chunk uploads only the reference frames of its own absolute indices and converts them on its card, so
            # device memory follows the chunk, not the clip.  The scratch is the worker's own (two workers on one card must not share one)
            sums = ref_sums.to(card) if n_ref == 1 else None
            state = {"scratch": None}
            def run(frames, first):
                # one library call per chunk: (the reference frames' statistics,) statistics, parameters and the apply pass (which
                # starts from the stored Lab f-planes for fp32 frames instead of repeating the forward transform)
                if n_ref == 1:
                    out, state["scratch"] = ops.chain_cm_apply(frames, d, sums, scratch=state["scratch"])
                    return out
                refs = upload(reference_image[first:first + frames.shape[0]], card).to(frames.dtype)
                out, state["scratch"] = ops.chain_cm_apply_refs(frames, d, refs, scratch=state["scratch"])
                return out
            return run
        devs = devices_from_env() if images.device.type == "cpu" else None
        out = run_frames(images, make_fn, batch_size, result_device(images), dev, devs)
        return (out,)


class _StencilNode:
    OP_CPU = nv.STENCIL_NONE
    OP_GPU = nv.STENCIL_NONE

    def _apply(self, images, strength, use_gpu):
        # RGB or RGBA: the reference's NumPy paths pad H and W only and filter every channel, and its avg_pool2d unsharp is per
        # channel too; its conv2d paths (Laplacian / Sobel with use_gpu) have groups=3 and reject 4 channels, so these do here.
        images = _as_frames(images, channels=(3, 4))
        op = self.OP_GPU if use_gpu else self.OP_CPU
        if images.shape[-1] == 4 and op in (nv.STENCIL_LAPLACIAN_GPU, nv.STENCIL_SOBEL_GPU):
            raise ValueError("%s with use_gpu=True takes 3-channel images (the torch path convolves with groups=3), got 4 channels"
                             % type(self).__name__)
        # use_gpu=False -> the numpy path's semantics (edge-replicated border); True -> the torch path's (zero padding).
        border = nv.BORDER_ZERO if use_gpu else nv.BORDER_REPLICATE
        s = float(strength)
        def run(frames, first):
            return ops.stencil3x3(frames, op, s, border)
        devs = devices_from_env() if images.device.type == "cpu" else None
        out = run_frames(images, lambda dev: run, 8, result_device(images, numpy_path=not use_gpu), compute_device(images), devs)
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

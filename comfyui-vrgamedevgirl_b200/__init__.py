"""comfyui-vrgamedevgirl_b200 — H100-native (sm_90a) implementation of the per-pixel video post-processing
hot path of the comfyui-vrgamedevgirl node pack, behind the same ComfyUI node API.

ComfyUI loads this directory as a custom node package and reads NODE_CLASS_MAPPINGS /
NODE_DISPLAY_NAME_MAPPINGS (reference plugin boundary: __init__.py:99-111,171-177).  Outside ComfyUI import it
with importlib.import_module("comfyui-vrgamedevgirl_b200") (the directory name is not a Python identifier).
"""
from . import _native, chain, ops  # noqa: F401
from .filter_nodes import (  # noqa: F401
    ColorMatchToReference,
    FastFilmGrain,
    FastLaplacianSharpen,
    FastSobelSharpen,
    FastUnsharpSharpen,
)
from .lut_nodes import VRGDG_LUTS, VRGDG_MakeLUT  # noqa: F401
from . import chain_nodes as _chain_nodes

__version__ = "0.1.0"

# keys and display names: nodes.py:1882-1886,1908-1912 and VRGDG_IV_Adjustments.py:426-434
NODE_CLASS_MAPPINGS = {
    "FastFilmGrain": FastFilmGrain,
    "ColorMatchToReference": ColorMatchToReference,
    "FastUnsharpSharpen": FastUnsharpSharpen,
    "FastLaplacianSharpen": FastLaplacianSharpen,
    "FastSobelSharpen": FastSobelSharpen,
    "VRGDG_LUTS": VRGDG_LUTS,
    "VRGDG_MakeLUT": VRGDG_MakeLUT,
}

NODE_DISPLAY_NAME_MAPPINGS = {
    "FastFilmGrain": "\U0001F39E\uFE0F Fast Film Grain",
    "ColorMatchToReference": "\U0001F3A8 Color Match To Reference",
    "FastUnsharpSharpen": "\U0001F3AF Fast Unsharp Sharpen",
    "FastLaplacianSharpen": "\U0001F300 Fast Laplacian Sharpen",
    "FastSobelSharpen": "\U0001F4CF Fast Sobel Sharpen",
    "VRGDG_LUTS": "VRGDG_LUTS",
    "VRGDG_MakeLUT": "VRGDG_MakeLUT",
}

# graph-reachable entries to the fused kernels and the video-enhance tensor path: two reference keys
# (VRGDG_VideoEnhanceNodes.py:422-437, VRGDG_StandaloneVideoEnhancerNodes.py:897-903) and two extra keys of this package
NODE_CLASS_MAPPINGS.update(_chain_nodes.NODE_CLASS_MAPPINGS)
NODE_DISPLAY_NAME_MAPPINGS.update(_chain_nodes.NODE_DISPLAY_NAME_MAPPINGS)

__all__ = ["NODE_CLASS_MAPPINGS", "NODE_DISPLAY_NAME_MAPPINGS"]

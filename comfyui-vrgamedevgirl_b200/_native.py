"""ctypes binding of libvrgdg_b200.so (C ABI: include/vrgdg_b200.h).

There is deliberately no fallback: if the library is missing, was built for another architecture, or no
CUDA device is visible, every operation raises.  The filters exist only as sm_90a kernels.
"""
import ctypes
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("VRGDG_B200_LIB") or os.path.join(_HERE, "lib", "libvrgdg_b200.so")   # env override: build experiments only

VRGDG_OK = 0
E_INVALID, E_UNSUPPORTED, E_CUDA, E_ALIGN = -1, -2, -3, -4

F32, F16, BF16, U8BGR = 0, 1, 2, 3
DTYPE_CODE = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16, torch.uint8: U8BGR}

STENCIL_NONE, STENCIL_BOX_UNSHARP, STENCIL_LAPLACIAN_CPU, STENCIL_LAPLACIAN_GPU, STENCIL_SOBEL_CPU, STENCIL_SOBEL_GPU = range(6)
BORDER_REPLICATE, BORDER_ZERO = 0, 1
SEED_PER_CLIP, SEED_PER_FRAME = 0, 1
CHAIN_FAST_MATH = 1
CHAIN_CM_RECOMPUTE = 2
CHAIN_CM_SERIAL = 4


class ChainDesc(ctypes.Structure):
    """struct vrgdg_chain_desc (include/vrgdg_b200.h)."""

    _fields_ = [
        ("grain_enabled", ctypes.c_int32),
        ("grain_intensity", ctypes.c_float),
        ("grain_sat", ctypes.c_float),
        ("grain_one_minus_sat", ctypes.c_float),
        ("grain_seed", ctypes.c_uint64),
        ("grain_frame0", ctypes.c_int64),
        ("grain_seed_mode", ctypes.c_int32),
        ("colormatch_enabled", ctypes.c_int32),
        ("cm_params", ctypes.c_void_p),
        ("cm_t", ctypes.c_float),
        ("cm_one_minus_t", ctypes.c_float),
        ("lut_enabled", ctypes.c_int32),
        ("lut", ctypes.c_void_p),
        ("lut_size", ctypes.c_int32),
        ("lut_dmin", ctypes.c_float * 3),
        ("lut_dspan", ctypes.c_float * 3),
        ("lut_blend", ctypes.c_float),
        ("lut_one_minus_blend", ctypes.c_float),
        ("stencil_op", ctypes.c_int32),
        ("stencil_strength", ctypes.c_float),
        ("stencil_border", ctypes.c_int32),
        ("post_grain_enabled", ctypes.c_int32),
        ("post_intensity", ctypes.c_float),
        ("post_sat", ctypes.c_float),
        ("post_one_minus_sat", ctypes.c_float),
        ("post_seed", ctypes.c_uint64),
        ("post_frame0", ctypes.c_int64),
        ("post_seed_mode", ctypes.c_int32),
    ]


class AdjustDesc(ctypes.Structure):
    """struct vrgdg_adjust_desc (include/vrgdg_b200.h)."""

    _fields_ = [
        ("enabled", ctypes.c_int32),
        ("offset_rgb", ctypes.c_float * 3),
        ("exposure", ctypes.c_float), ("contrast", ctypes.c_float), ("saturation", ctypes.c_float),
        ("highlights", ctypes.c_float), ("shadows", ctypes.c_float), ("whites", ctypes.c_float), ("blacks", ctypes.c_float),
        ("clarity_on", ctypes.c_int32), ("sharpen_on", ctypes.c_int32), ("blur_kernel", ctypes.c_int32),
        ("clarity", ctypes.c_float), ("sharpen", ctypes.c_float),
        ("fade_on", ctypes.c_int32), ("vignette_on", ctypes.c_int32),
        ("fade_mul", ctypes.c_float), ("fade_add", ctypes.c_float), ("vignette", ctypes.c_float),
    ]


class ResizeDesc(ctypes.Structure):
    """struct vrgdg_resize_desc (include/vrgdg_b200.h)."""

    _fields_ = [
        ("mode", ctypes.c_int32),
        ("src_x0", ctypes.c_int32), ("src_y0", ctypes.c_int32), ("src_w", ctypes.c_int32), ("src_h", ctypes.c_int32),
        ("res_w", ctypes.c_int32), ("res_h", ctypes.c_int32),
        ("off_x", ctypes.c_int32), ("off_y", ctypes.c_int32),
    ]


_vp, _i, _i64, _u64, _f = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_uint64, ctypes.c_float
_fp = ctypes.POINTER(ctypes.c_float)

# name -> (restype, argtypes); must list every symbol include/vrgdg_b200.h declares
SIGNATURES = {
    "vrgdg_version": (_i, []),
    "vrgdg_last_error": (ctypes.c_char_p, []),
    "vrgdg_device_info": (_i, [ctypes.POINTER(_i)] * 3),
    "vrgdg_launch_count": (_i64, []),
    "vrgdg_last_tile_path": (ctypes.c_char_p, []),
    "vrgdg_lut3d_packed_bytes": (_i64, [_i]),
    "vrgdg_lut3d_pack": (_i, [_vp, _vp, _i, _vp]),
    "vrgdg_lut3d_apply": (_i, [_vp, _vp, _i64, _i, _i, _vp, _i, _fp, _fp, _f, _f, _vp]),
    "vrgdg_grain": (_i, [_vp, _vp, _i, _i, _i, _i, _f, _f, _f, _u64, _i64, _i, _vp, _vp]),
    "vrgdg_grain_noise": (_i, [_vp, _i, _i, _i, _u64, _i64, _i, _vp]),
    "vrgdg_stencil3x3": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp]),
    "vrgdg_lab_moments_scratch_bytes": (_i64, [_i]),
    "vrgdg_lab_moments": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i64, _vp]),
    "vrgdg_colormatch_params": (_i, [_vp, _i, _vp, _i, _vp, _vp]),
    "vrgdg_colormatch_apply": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _f, _f, _vp]),
    "vrgdg_chain_apply": (_i, [_vp, _vp, _i, _i, _i, _i, ctypes.POINTER(ChainDesc), _vp]),
    "vrgdg_chain_apply_ext": (_i, [_vp, _vp, _i, _i, _i, _i, ctypes.POINTER(ChainDesc), _vp, _i, _vp]),
    "vrgdg_chain_lab_moments": (_i, [_vp, _i, _i, _i, _i, ctypes.POINTER(ChainDesc), _vp, _vp, _i64, _vp]),
    "vrgdg_chain_lab_moments_ext": (_i, [_vp, _i, _i, _i, _i, ctypes.POINTER(ChainDesc), _vp, _vp, _vp, _i64, _vp]),
    "vrgdg_chain_cm_scratch_bytes": (_i64, [_i, _i, _i, _i, _i, _i]),
    "vrgdg_chain_cm_apply": (_i, [_vp, _vp, _i, _i, _i, _i, ctypes.POINTER(ChainDesc), _vp, _i, _vp, _i, _vp, _i64, _i, _vp]),
    "vrgdg_adjust_scratch_bytes": (_i64, [_i, _i, _i, ctypes.POINTER(AdjustDesc)]),
    "vrgdg_adjust": (_i, [_vp, _vp, _i, _i, _i, _i, ctypes.POINTER(AdjustDesc), _vp, _vp, _vp, _i64, _vp]),
    "vrgdg_resize": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, ctypes.POINTER(ResizeDesc), _vp]),
    "vrgdg_blend": (_i, [_vp, _vp, _vp, _i64, _i, _f, _f, _vp]),
    "vrgdg_hist_counts": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "vrgdg_histmatch_tables": (_i, [_vp, _i, _vp, _i, _vp, _vp]),
    "vrgdg_histmatch_apply": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _f, _f, _vp]),
    "vrgdg_temporal_sharpen": (_i, [_vp, _vp, _i, _i, _i, _i, _f, _vp, _vp, _vp]),
    "vrgdg_lanczos4_tables": (_i, [_i, _i, _vp, _vp]),
    "vrgdg_lanczos4_scratch_bytes": (_i64, [_i, _i, _i]),
    "vrgdg_lanczos4_resize_u8": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "vrgdg_u8bgr_to_rgb": (_i, [_vp, _vp, _i64, _i, _vp]),
    "vrgdg_rgb_to_u8bgr": (_i, [_vp, _vp, _i64, _i, _vp]),
}

_lib = None
_lock = threading.Lock()


def load_library():
    """dlopen the in-tree library and type its entry points.  Raises RuntimeError when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libvrgdg_b200.so is not built (%s). Run `python comfyui-vrgamedevgirl_b200/build.py` "
                "(needs nvcc; no GPU required to build). There is no CPU fallback for these nodes." % LIB_PATH
            )
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the .so is stale
            fn.restype = res
            fn.argtypes = args
        if lib.vrgdg_version() != 1:
            raise RuntimeError("libvrgdg_b200.so ABI version %d != 1; rebuild it" % lib.vrgdg_version())
        _lib = lib
    return _lib


def check(rc):
    """Map a VRGDG_E_* return code onto the exception type the reference raises for that class of error."""
    if rc == VRGDG_OK:
        return
    msg = load_library().vrgdg_last_error().decode("utf-8", "replace")
    if rc == E_CUDA:
        raise RuntimeError("vrgdg_b200: " + msg)
    raise ValueError("vrgdg_b200: " + msg)


def require_cuda(t, name="tensor"):
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if t.device.type != "cuda":
        raise RuntimeError("vrgdg_b200: %s must live on a CUDA device (got %s); the filters have no CPU path" % (name, t.device))
    if t.dtype not in DTYPE_CODE:
        raise ValueError("vrgdg_b200: unsupported dtype %s (float32 / float16 / bfloat16 / uint8 BGR)" % t.dtype)
    return t if t.is_contiguous() else t.contiguous()


def stream_ptr(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def launch_count():
    return int(load_library().vrgdg_launch_count())


def last_tile_path():
    return load_library().vrgdg_last_tile_path().decode()

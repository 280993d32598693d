"""The video-tools matrix: the adjust, resample, blend, 4-channel LUT and uint8 codec kernels that VRGDG_INSTANTIATE builds for
every frame dtype, the cases tests/test_gpu_video_tools_matrix.py runs against the oracle, the error bar of each case, and a mirror of
how vrgdg_inst.cuh / vrgdg_adjust.cuh pick the kernel for a case.  No GPU and no torch needed here, so the CPU suite can check that
the matrix reaches every instantiation (tests/test_video_tools_matrix_coverage.py)."""
import itertools
import json
import os
import re
from collections import namedtuple

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "comfyui-vrgamedevgirl_b200", "csrc")
META = os.path.join(ROOT, "tests", "golden", "reference_meta.json")

DTYPES = ("f32", "f16", "bf16", "u8")
FLOAT_DTYPES = ("f32", "f16", "bf16")
ULP = {"f16": 2.0 ** -11, "bf16": 2.0 ** -8}                        # spacing of the 16-bit type in [0.5, 1)
CTYPE = {"float": "f32", "__half": "f16", "__nv_bfloat16": "bf16", "uint8_t": "u8"}


# ---- adjust (_apply_adjust_tensor) ------------------------------------------------------------------------------------------
def _golden_adjust():
    with open(META, encoding="utf-8") as fh:
        return json.load(fh)["adjust_cases"]


_G = _golden_adjust()
ADJUST_SETTINGS = {
    "pointwise": _G["pointwise"],                                    # stage A only: k_adjust_point
    "fade_vignette": _G["fade_vignette"],                            # stages A + D in the point kernel (vignette mask)
    "clarity": _G["clarity"],                                        # k x k reflect box, last pass
    "sharpen": _G["sharpen"],                                        # 3 x 3 replicate box, last pass
    "clarity_sharpen": {"clarity": 45, "sharpen": 50, "exposure": 5},  # clarity into the second scratch frame, then sharpen
    "everything": _G["everything"],                                  # every stage, vignette included
    "disabled": _G["disabled"],                                      # clamp only
}

# (B, H, W): the small side selects the clarity window K (k = min(9, odd H, odd W), < 3 -> 1) and sits first as H, then as W;
# W % 4 == 0 takes the 4-pixel vector stores, W % 4 != 0 the scalar ones.  Tiles are 16 rows x 64 pixels, so every shape with
# W > 64 spans two tile columns; "k9_tiles*" are 3 x 3 tiles whose last row and column are partial.
ADJUST_SHAPES = {
    "k1_h1": (2, 1, 68), "k1_h2": (2, 2, 37), "k1_w1": (2, 40, 1), "k1_w2": (2, 45, 2),
    "k3_h3": (2, 3, 72), "k3_h4": (2, 4, 45), "k3_w3": (2, 37, 3), "k3_w4": (2, 33, 4),
    "k5_h5": (2, 5, 68), "k5_h6": (2, 6, 45), "k5_w5": (2, 37, 5), "k5_w6": (2, 35, 6),
    "k7_h7": (2, 7, 72), "k7_h8": (2, 8, 45), "k7_w7": (2, 37, 7), "k7_w8": (2, 33, 8),
    "k9_h9": (2, 9, 76), "k9_w9": (2, 70, 9),
    "k9_tiles": (2, 37, 140), "k9_tiles_ragged": (2, 35, 133),
}

AdjustCase = namedtuple("AdjustCase", "setting dtype shape")
ADJUST_CASES = [AdjustCase(s, d, sh) for s, d, sh in itertools.product(ADJUST_SETTINGS, DTYPES, ADJUST_SHAPES)]


def adjust_id(c):
    return "adjust-%s-%s-%s" % (c.setting, c.dtype, c.shape)


def blur_kernel(H, W):
    """video_tools._adjust_desc: the clarity window (1 means the reference's blur returns its input)"""
    k = min(9, H if H % 2 else H - 1, W if W % 2 else W - 1)
    return k if k >= 3 else 1


def _scaled(st, key):
    try:
        return float(st.get(key, 0.0)) / 100.0
    except (TypeError, ValueError):
        return 0.0


def adjust_kernels(c):
    """{(kernel, dtype, ...)} launch_adjust runs for a case: ("point", dtype, TO_SCRATCH) and ("box", dtype, K, MODE, LAST, store)"""
    st = ADJUST_SETTINGS[c.setting]
    B, H, W = ADJUST_SHAPES[c.shape]
    enabled = st.get("enabled", True) is not False
    C = enabled and abs(_scaled(st, "clarity")) > 0.001
    S = enabled and _scaled(st, "sharpen") > 0.001
    store = "vec" if W % 4 == 0 else "scalar"
    if not (C or S):
        return {("point", c.dtype, False)}
    out = {("point", c.dtype, True)}
    if C:
        out.add(("box", c.dtype, blur_kernel(H, W), 0, not S, store))
    if S:
        out.add(("box", c.dtype, 3, 1, True, store))
    return out


# ---- resize (_resize_batch / _restore_batch) ----------------------------------------------------------------------------------
RESIZE_MODES = ("nearest", "bilinear", "bicubic", "area")
METHOD = {"nearest": "Nearest", "bilinear": "Bilinear", "bicubic": "Bicubic (recommended)", "area": "Area"}
RESIZE_SRC = (2, 37, 53)
# geometry -> (fit mode, target width, target height); "restore" resamples the letterboxed 80 x 80 frame (content rows 12 .. 67)
# back to 53 x 37, "roi" is a window that starts at (5, 7) and stops short of the frame's right and bottom edges
RESIZE_GEOMETRIES = {
    "stretch": ("Stretch to dimensions", 90, 29),
    "crop": ("Crop to fill", 64, 64),                                # resampled 92 x 64 at offset -14 (negative placement)
    "letterbox": ("Fit with letterbox (preserve all)", 80, 80),    # resampled 80 x 56 at offset +12
    "restore": ("Fit with letterbox (preserve all)", 53, 37),
    "roi": ("Stretch to dimensions", 61, 33),
}
ROI = (5, 7, 40, 25)                                                 # x0, y0, w, h inside RESIZE_SRC

# (source, resampled) sizes along one axis where the area window's o*in passes 2^24: an fp32 quotient there picks the wrong window
# (4007 -> 5009 even reads one pixel past the ROI), ATen's integer bounds do not.  Each runs as a [1, 2, W, 3] strip (x) and a
# [1, H, 2, 3] strip (y) whose ROI stops one pixel short of the frame edge.
AREA_STRIPS = ((4007, 5009), (4021, 6032), (7679, 3840), (4319, 4320), (5119, 5120), (6143, 3072))
STRIP_MODES = ("nearest", "area")

ResizeCase = namedtuple("ResizeCase", "mode dtype channels geometry")


def build_resize_cases():
    cases = [ResizeCase(m, d, ch, g) for m, d, ch, g in itertools.product(RESIZE_MODES, FLOAT_DTYPES, (3, 4), RESIZE_GEOMETRIES)]
    for m, d, axis, (src, dst) in itertools.product(STRIP_MODES, FLOAT_DTYPES, ("x", "y"), AREA_STRIPS):
        cases.append(ResizeCase(m, d, 3, "strip-%s-%d-%d" % (axis, src, dst)))
    return cases


RESIZE_CASES = build_resize_cases()


def resize_id(c):
    return "resize-%s-%s-c%d-%s" % (c.mode, c.dtype, c.channels, c.geometry)


def strip_of(c):
    """(axis, source, resampled) of a strip case, or None"""
    if not c.geometry.startswith("strip-"):
        return None
    _, axis, src, dst = c.geometry.split("-")
    return axis, int(src), int(dst)


def area_bounds(o, n_in, n_out):
    """ATen's adaptive-average window [start, end) of output index o: floor(o*in/out), ceil((o+1)*in/out) in integers"""
    return (o * n_in) // n_out, ((o + 1) * n_in + n_out - 1) // n_out


# ---- blend, 4-channel LUT, codecs ---------------------------------------------------------------------------------------------
BLEND_WEIGHTS = {"orig": 0.0, "restored": 1.0, "s035": 0.35}         # strength s: originals * (1 - s) + restored * s
BLEND_SHAPE = (3, 7, 11, 3)                                          # 693 elements: not a multiple of 4 or 8
BlendCase = namedtuple("BlendCase", "dtype weights")
BLEND_CASES = [BlendCase(d, w) for d, w in itertools.product(FLOAT_DTYPES, BLEND_WEIGHTS)]

LUT_STRENGTHS = {"b1": 10.0, "b035": 3.5}                            # blend = strength / 10
LUT_DOMAIN = ((-0.125, 0.0625, 0.0), (1.125, 0.9375, 0.75))          # non-unit, exact in every float dtype
LutCase = namedtuple("LutCase", "dtype strength")
LUT_RGBA_CASES = [LutCase(d, s) for d, s in itertools.product(FLOAT_DTYPES, LUT_STRENGTHS)]

CODEC_DIRECTIONS = ("to_float", "to_u8")
CodecCase = namedtuple("CodecCase", "dtype direction")
CODEC_CASES = [CodecCase(d, k) for d, k in itertools.product(FLOAT_DTYPES, CODEC_DIRECTIONS)]

# vrgdg_lut3d_apply walks a 3-channel pixel stream in launches of 2^30 pixels; 4097 more make a second, odd-sized launch (scalar path)
LUT_STREAM_CHUNK = 1 << 30
LUT_STREAM_PIXELS = LUT_STREAM_CHUNK + 4097


# ---- error bars ---------------------------------------------------------------------------------------------------------------
# max |kernel - oracle| per case; 16-bit frames against the oracle on the up-cast input rounded once to the frame dtype, uint8 frames
# as bytes (frames_to_tensor -> op -> tensor_to_frames):
#   adjust, every stage and dtype (vignette: oracle with a correctly rounded sqrt, as the kernel's __fsqrt_rn)   0 (torch.equal)
#   resize nearest / area, every dtype                                                                          0
#   resize bilinear / bicubic: fp32 (ATen's CPU kernels associate differently between thread counts)            2e-6
#   resize bilinear / bicubic: fp16 / bf16 (two roundings of values 2e-6 apart)                                 one spacing of the type
#   blend, 4-channel LUT (alpha bit for bit at blend 1), codecs, the LUT stream past 2^30 pixels                0
BAR_RESIZE_F32 = 2e-6


def resize_bar(c):
    if c.mode in ("nearest", "area"):
        return 0.0
    return BAR_RESIZE_F32 if c.dtype == "f32" else ULP[c.dtype]


# ---- what the sources build ---------------------------------------------------------------------------------------------------
def _read(name):
    with open(os.path.join(CSRC, name), encoding="utf-8") as fh:
        return fh.read()


def _function_body(src, signature):
    """text of the function whose definition starts with `signature`, up to its closing brace at column 0"""
    i = src.find(signature)
    assert i >= 0, "no %r" % signature
    j = src.find("\n}\n", i)
    assert j > i, "no end of %r" % signature
    return src[i:j]


def instantiated_dtypes(macro):
    """frame dtypes whose translation unit expands VRGDG_INSTANTIATE / VRGDG_INSTANTIATE_CODECS"""
    out = set()
    for unit in ("vrgdg_f32.cu", "vrgdg_f16.cu", "vrgdg_bf16.cu", "vrgdg_u8.cu"):
        for t in re.findall(r"^%s\((\w+)\)" % macro, _read(unit), re.M):
            out.add(CTYPE[t])
    return out


def adjust_instantiations():
    """{("point", dtype, TO_SCRATCH)} | {("box", dtype, K, MODE, LAST, store)} that launch_adjust can reach: every K of the
    launch_adjust_box switch for a call that passes the descriptor's window, only the named K for a call with a literal, both stores"""
    src = _read("vrgdg_adjust.cuh")
    sw = _function_body(src, "template <typename T, int MODE, bool LAST>\ncudaError_t launch_adjust_box(")
    switch = {}
    for label, k in re.findall(r"(case \d+|default): k_adjust_box<T, MODE, LAST, (\d+)>", sw):
        switch["default" if label == "default" else int(label.split()[1])] = int(k)
    assert "default" in switch, "launch_adjust_box has no default window"
    la = _function_body(src, "template <typename T>\ncudaError_t launch_adjust(")
    calls = re.findall(r"launch_adjust_box<T, (\d), (true|false)>\(([^,]+),", la)
    points = re.findall(r"k_adjust_point<T, (true|false)>", la)
    assert calls and points, "launch_adjust calls no kernel"
    out = set()
    for dt in instantiated_dtypes("VRGDG_INSTANTIATE"):
        for p in points:
            out.add(("point", dt, p == "true"))
        for mode, last, karg in calls:
            karg = karg.strip()
            ks = {switch.get(int(karg), switch["default"])} if re.fullmatch(r"\d+", karg) else set(switch.values())
            for k, store in itertools.product(ks, ("vec", "scalar")):
                out.add(("box", dt, k, int(mode), last == "true", store))
    return out


def resize_modes():
    """modes of the launch_resize switch (the default label is the area kernel)"""
    body = _function_body(_read("vrgdg_resize.cuh"), "template <typename T>\ncudaError_t launch_resize(")
    modes = set(m.lower() for m in re.findall(r"k_resize<T, VRGDG_RESIZE_(\w+)>", body))
    assert "default: k_resize<T, VRGDG_RESIZE_AREA>" in body
    return modes


def _abi_body(fn):
    return _function_body(_read("vrgdg_abi.cu"), "int %s(" % fn)


def resize_instantiations():
    """{(dtype, mode, channels)}: the ABI takes float frames only, 3 or 4 channels"""
    body = _abi_body("vrgdg_resize")
    assert "dtype == VRGDG_U8BGR) return fail" in body and "channels != 3 && channels != 4" in body
    dts = instantiated_dtypes("VRGDG_INSTANTIATE") - {"u8"}
    return set(itertools.product(dts, resize_modes(), (3, 4)))


def blend_dtypes():
    assert "dtype == VRGDG_U8BGR) return fail" in _abi_body("vrgdg_blend")
    return instantiated_dtypes("VRGDG_INSTANTIATE") - {"u8"}


def lut_rgba_dtypes():
    """launch_lut_rgba runs for 4-channel frames; the ABI refuses 4-channel uint8"""
    assert "channels == 4 && dtype == VRGDG_U8BGR) return fail" in _abi_body("vrgdg_lut3d_apply")
    return instantiated_dtypes("VRGDG_INSTANTIATE") - {"u8"}


def codec_dtypes():
    return instantiated_dtypes("VRGDG_INSTANTIATE_CODECS")

"""VRGDG_LUTS / VRGDG_MakeLUT (reference: VRGDG_IV_Adjustments.py) with the trilinear sampler on sm_90a.

Host-side pieces (.cube text parsing, palette-LUT construction, file naming, cache keys) keep the
reference's semantics; the per-pixel work (normalise, cell lookup, 8-corner trilinear blend, strength blend)
is vrgdg_lut3d_apply in libvrgdg_b200.so and is bit-identical to the reference's CPU result for fp32 images.
"""
import os

import numpy as np
import torch

from . import ops
from ._runtime import compute_device, devices_from_env, run_frames

LUTS_DIR = os.path.join(os.path.dirname(__file__), "LUTS")
SUPPORTED_LUT_EXTENSIONS = (".cube",)
NO_LUTS = "No LUT files found"            # sentinel, VRGDG_IV_Adjustments.py:27,36

# basic colour names accepted by the palette parser (:9-22)
NAMED_COLORS = dict(
    black="#000000", white="#ffffff", red="#ff0000", green="#00ff00", blue="#0000ff", yellow="#ffff00", cyan="#00ffff",
    magenta="#ff00ff", orange="#ffa500", purple="#800080", pink="#ffc0cb", teal="#008080",
)


def _list_lut_files():
    """:25-36 — case-insensitively sorted *.cube names, or the sentinel."""
    if not os.path.isdir(LUTS_DIR):
        return [NO_LUTS]
    names = sorted(
        (n for n in os.listdir(LUTS_DIR) if n.lower().endswith(SUPPORTED_LUT_EXTENSIONS) and os.path.isfile(os.path.join(LUTS_DIR, n))),
        key=str.lower,
    )
    return names or [NO_LUTS]


def _sanitize_filename_part(value):
    """:39-42"""
    text = str(value or "").strip().lower()
    pieces = "".join(c if c.isalnum() else "_" for c in text).split("_")
    return "_".join(p for p in pieces if p) or "custom"


def _parse_hex_color(token):
    """:45-65"""
    token = str(token or "").strip().lower()
    token = NAMED_COLORS.get(token, token)
    if token.startswith("#"):
        token = token[1:]
    if len(token) == 3:
        token = "".join(c + c for c in token)
    if len(token) != 6 or any(c not in "0123456789abcdef" for c in token):
        raise ValueError(f"Invalid color '{token}'. Use hex like #ff8800 or a basic color name.")
    return np.array([int(token[i:i + 2], 16) / 255.0 for i in (0, 2, 4)], dtype=np.float32)


def _parse_color_list(colors_text):
    """:68-72"""
    items = [p.strip() for p in str(colors_text or "").split(",") if p.strip()]
    if not items:
        raise ValueError("Provide one or more colors separated by commas.")
    return np.stack([_parse_hex_color(p) for p in items], axis=0)


def _build_palette_lut(colors_text, lut_size):
    """:75-105 — luma ramp through the palette, luma-preserving rescale, 0.82/0.18 chroma mix.  float32 numpy,
    same operation order as the reference so the generated table is identical."""
    palette = _parse_color_list(colors_text)
    axis = np.linspace(0.0, 1.0, int(lut_size), dtype=np.float32)
    blue, green, red = np.meshgrid(axis, axis, axis, indexing="ij")
    source = np.stack([red, green, blue], axis=-1)
    luma = (0.2126 * source[..., 0]) + (0.7152 * source[..., 1]) + (0.0722 * source[..., 2])

    if palette.shape[0] == 1:
        target = np.empty(luma.shape + (3,), dtype=np.float32)
        target[...] = palette[0]
    else:
        knots = np.linspace(0.0, 1.0, palette.shape[0], dtype=np.float32)
        flat = luma.reshape(-1)
        ramp = np.stack([np.interp(flat, knots, palette[:, c]) for c in range(3)], axis=-1)
        target = ramp.reshape(luma.shape + (3,)).astype(np.float32)

    target_luma = (0.2126 * target[..., 0]) + (0.7152 * target[..., 1]) + (0.0722 * target[..., 2])
    gain = luma / np.maximum(target_luma, 1e-6)
    target = np.clip(target * gain[..., None], 0.0, 1.0)
    chroma = source - luma[..., None]
    table = np.clip((target * 0.82) + ((target + chroma) * 0.18), 0.0, 1.0)
    return torch.from_numpy(table.astype(np.float32))


def _write_cube_file(lut_tensor, lut_path):
    """:108-123 — TITLE, size, unit domain, '%.6f' triples with red fastest."""
    size = int(lut_tensor.shape[0])
    table = lut_tensor.detach().cpu().numpy().reshape(-1, 3)
    os.makedirs(os.path.dirname(lut_path), exist_ok=True)
    with open(lut_path, "w", encoding="utf-8") as fh:
        fh.write(f'TITLE "{os.path.basename(lut_path)}"\n')
        fh.write(f"LUT_3D_SIZE {size}\n")
        fh.write("DOMAIN_MIN 0.0 0.0 0.0\n")
        fh.write("DOMAIN_MAX 1.0 1.0 1.0\n")
        fh.writelines(f"{r:.6f} {g:.6f} {b:.6f}\n" for r, g, b in table)


def _next_available_lut_path(base_name):
    """:126-137"""
    os.makedirs(LUTS_DIR, exist_ok=True)
    path = os.path.join(LUTS_DIR, f"{base_name}.cube")
    n = 2
    while os.path.exists(path):
        path = os.path.join(LUTS_DIR, f"{base_name}_{n}.cube")
        n += 1
    return path


def _blend_of(strength):
    """strength widget 0..10 -> blend 0..1 (:355)"""
    return max(0.0, min(10.0, float(strength))) / 10.0


def _run_lut(image, lut_data, strength):
    """Shared tail of apply_lut / create_and_apply (:347-361, :409-423) and _apply_lut_tensor
    (VRGDG_LUTVideoTools.py:172-185): returns a tensor on image.device."""
    if image.ndim != 4 or image.shape[-1] < 3:
        raise ValueError("VRGDG_LUTS expects IMAGE input shaped like [batch, height, width, channels].")
    if image.shape[-1] > 4:
        raise ValueError("vrgdg_b200: IMAGE tensors with more than 4 channels are not supported")
    blend = _blend_of(strength)
    if blend <= 0.0:
        return image
    dev = compute_device(image)
    work = image if image.dtype in (torch.float32, torch.float16, torch.bfloat16) else image.float()
    # domain bounds are cast to the image dtype before the span clamp, as the reference does (:295,:351-352)
    dmin = lut_data["domain_min"].to(dtype=work.dtype)
    dmax = lut_data["domain_max"].to(dtype=work.dtype)
    span = torch.clamp(dmax - dmin, min=1e-6)
    lo, sp = dmin.float().tolist(), span.float().tolist()
    if work.device.type == "cuda":
        return ops.lut3d_apply(work.to(dev), _device_lut(lut_data, dev), lo, sp, blend, 1.0 - blend).to(device=image.device)

    # host frames: the three-stream pipeline of the other nodes (chunked upload / lookup / download, pinned result), sharded over the
    # VRGDG_DEVICES cards.  make_fn runs in the calling thread, so the packed-table cache is never written from a worker.
    def make_fn(card):
        lut_dev = _device_lut(lut_data, card)
        return lambda f, i: ops.lut3d_apply(f, lut_dev, lo, sp, blend, 1.0 - blend)
    return run_frames(work, make_fn, 0, image.device, dev, devices_from_env())


def _device_lut(lut_data, dev):
    cache = lut_data.setdefault("_device", {})
    key = str(dev)
    if key not in cache:
        cache[key] = ops.pack_lut(lut_data["lut"], dev)      # device layout, built once per (file version, device)
    return cache[key]


class VRGDG_LUTS:
    CATEGORY = "VRGDG/IV Adjustments"
    RETURN_TYPES = ("IMAGE",)
    RETURN_NAMES = ("image",)
    FUNCTION = "apply_lut"

    _LUT_CACHE = {}

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "image": ("IMAGE",),
                "lut_name": (_list_lut_files(),),
                "device": (["auto", "cuda", "cpu"], {"default": "auto"}),
                "strength": ("FLOAT", {"default": 10.0, "min": 0.0, "max": 10.0, "step": 0.1}),
            }
        }

    @classmethod
    def IS_CHANGED(cls, image, lut_name, device, strength):
        """:159-169"""
        if lut_name == NO_LUTS:
            return f"missing|{device}|{strength}"
        state = cls._get_luts_folder_state()
        path = os.path.join(LUTS_DIR, lut_name)
        if not os.path.isfile(path):
            return f"{state}|missing|{lut_name}|{device}|{strength}"
        return f"{state}|{lut_name}|{os.path.getmtime(path)}|{device}|{strength}"

    @staticmethod
    def _resolve_device(requested_device, image):
        """:171-185.  The widget only ever chose where the reference *computed*; results always return to
        image.device (:361).  Here the compute device is always CUDA: "cpu" is accepted for workflow
        compatibility and still computes on the GPU; without a GPU every choice raises."""
        requested = str(requested_device or "auto").strip().lower()
        if not torch.cuda.is_available():
            raise RuntimeError("VRGDG_LUTS: CUDA was selected, but CUDA is not available." if requested == "cuda"
                               else "VRGDG_LUTS (vrgdg_b200): CUDA is not available and this build has no CPU path.")
        return compute_device(image)

    @staticmethod
    def _get_luts_folder_state():
        """:187-201"""
        if not os.path.isdir(LUTS_DIR):
            return "missing"
        parts = []
        for name in _list_lut_files():
            if name == NO_LUTS:
                continue
            path = os.path.join(LUTS_DIR, name)
            try:
                parts.append(f"{name}:{os.path.getmtime(path)}:{os.path.getsize(path)}")
            except OSError:
                parts.append(f"{name}:missing")
        return "|".join(parts) if parts else "empty"

    @classmethod
    def _load_lut(cls, lut_name):
        """:203-219 — one-entry cache keyed by (path, mtime, size); also holds the device copy."""
        if lut_name == NO_LUTS:
            raise ValueError("No LUT files were found in the LUTS folder.")
        path = os.path.join(LUTS_DIR, lut_name)
        if not os.path.isfile(path):
            raise FileNotFoundError(f"LUT file not found: {path}")
        key = (path, os.path.getmtime(path), os.path.getsize(path))
        hit = cls._LUT_CACHE.get(key)
        if hit is None:
            hit = cls._parse_cube_file(path)
            cls._LUT_CACHE = {key: hit}
        return hit

    @staticmethod
    def _parse_cube_file(lut_path):
        """:222-282 — .cube text -> [S,S,S,3] float32 in [blue][green][red][rgb] order."""
        size = None
        bounds = {"DOMAIN_MIN": np.array([0.0, 0.0, 0.0], dtype=np.float32), "DOMAIN_MAX": np.array([1.0, 1.0, 1.0], dtype=np.float32)}
        values = []
        with open(lut_path, "r", encoding="utf-8", errors="ignore") as fh:
            for raw in fh:
                line = raw.strip()
                if not line or line[0] == "#":
                    continue
                head = line.upper()
                if head.startswith("TITLE "):
                    continue
                if head.startswith("LUT_1D_SIZE"):
                    raise ValueError(f"1D LUTs are not supported: {os.path.basename(lut_path)}")
                fields = line.split()
                if head.startswith("LUT_3D_SIZE"):
                    if len(fields) != 2:
                        raise ValueError(f"Invalid LUT_3D_SIZE line in {lut_path}")
                    size = int(fields[1])
                    continue
                keyword = next((k for k in bounds if head.startswith(k)), None)
                if keyword is not None:
                    if len(fields) != 4:
                        raise ValueError(f"Invalid {keyword} line in {lut_path}")
                    bounds[keyword] = np.array([float(v) for v in fields[1:4]], dtype=np.float32)
                    continue
                if len(fields) == 3:           # anything else that is not a triple is skipped silently
                    values.extend(float(v) for v in fields)
        if size is None:
            raise ValueError(f"Missing LUT_3D_SIZE in {lut_path}")
        expected = size * size * size * 3
        if len(values) != expected:
            raise ValueError(f"Invalid LUT data length in {lut_path}. Expected {expected} floats, got {len(values)}.")
        table = np.asarray(values, dtype=np.float32).reshape(size, size, size, 3)   # red fastest -> [b][g][r][rgb]
        return {
            "size": size,
            "lut": torch.from_numpy(table),
            "domain_min": torch.from_numpy(bounds["DOMAIN_MIN"]),
            "domain_max": torch.from_numpy(bounds["DOMAIN_MAX"]),
        }

    @classmethod
    def _apply_cube_lut(cls, image, lut_tensor, domain_min, domain_max):
        """:288-343 — trilinear sample without the strength blend; image must already be on a CUDA device."""
        if image.ndim != 4 or image.shape[-1] < 3:
            raise ValueError("VRGDG_LUTS expects IMAGE input shaped like [batch, height, width, channels].")
        span = torch.clamp(domain_max - domain_min, min=1e-6)
        return ops.lut3d_apply(image, ops.pack_lut(lut_tensor, image.device), domain_min.float().tolist(), span.float().tolist(), 1.0, 0.0)

    def apply_lut(self, image, lut_name, device, strength):
        """:345-361"""
        lut_data = self._load_lut(lut_name)
        self._resolve_device(device, image)
        return (_run_lut(image, lut_data, strength),)


class VRGDG_MakeLUT:
    CATEGORY = "VRGDG/IV Adjustments"
    RETURN_TYPES = ("IMAGE", "STRING", "STRING")
    RETURN_NAMES = ("image", "lut_name", "lut_path")
    FUNCTION = "create_and_apply"

    @classmethod
    def INPUT_TYPES(cls):
        return {
            "required": {
                "image": ("IMAGE",),
                "colors": ("STRING", {"default": "#0b1d51, #1f6aa5, #f3d27a", "multiline": False}),
                "name_suffix": ("STRING", {"default": "palette", "multiline": False}),
                "lut_size": ("INT", {"default": 33, "min": 8, "max": 128, "step": 1}),
                "device": (["auto", "cuda", "cpu"], {"default": "auto"}),
                "strength": ("FLOAT", {"default": 10.0, "min": 0.0, "max": 10.0, "step": 0.1}),
            }
        }

    @classmethod
    def IS_CHANGED(cls, image, colors, name_suffix, lut_size, device, strength):
        return f"{colors}|{name_suffix}|{lut_size}|{device}|{strength}"

    def create_and_apply(self, image, colors, name_suffix, lut_size, device, strength):
        """:393-423 — build the palette LUT, save it next to the shipped ones, apply it."""
        table = _build_palette_lut(colors, lut_size)
        color_slug = "_".join(_sanitize_filename_part(p) for p in str(colors).split(",") if p.strip())
        suffix_slug = _sanitize_filename_part(name_suffix)
        base = f"{color_slug}_{suffix_slug}" if suffix_slug else color_slug
        lut_path = _next_available_lut_path(base)
        _write_cube_file(table, lut_path)
        lut_data = {
            "size": int(table.shape[0]),
            "lut": table,
            "domain_min": torch.tensor([0.0, 0.0, 0.0], dtype=torch.float32),
            "domain_max": torch.tensor([1.0, 1.0, 1.0], dtype=torch.float32),
        }
        VRGDG_LUTS._resolve_device(device, image)
        return (_run_lut(image, lut_data, strength), os.path.basename(lut_path), lut_path)


NODE_CLASS_MAPPINGS = {"VRGDG_LUTS": VRGDG_LUTS, "VRGDG_MakeLUT": VRGDG_MakeLUT}
NODE_DISPLAY_NAME_MAPPINGS = {"VRGDG_LUTS": "VRGDG_LUTS", "VRGDG_MakeLUT": "VRGDG_MakeLUT"}

"""Tensor-level wrappers over the C ABI: CUDA tensors in, CUDA tensors out, work enqueued on the
caller's current stream.  Python allocates every output (torch's allocator owns frame memory)."""
import ctypes

import numpy as np
import torch

from . import _native as nv


def _frames(images, name="images"):
    t = nv.require_cuda(images, name)
    if t.ndim != 4 or t.shape[-1] != 3:
        raise ValueError("vrgdg_b200: %s must be shaped [batch, height, width, 3], got %s" % (name, tuple(t.shape)))
    return t


def _f32(v):
    return ctypes.c_float(float(v))


def _noise(ext_noise, frames):
    """external N(0,1) tensor: same shape/device as the frames, same dtype (float32 for uint8 frames), RGB order"""
    n = nv.require_cuda(ext_noise, "ext_noise")
    want = torch.float32 if frames.dtype == torch.uint8 else frames.dtype
    if n.shape != frames.shape or n.dtype != want or n.device != frames.device:
        raise ValueError("vrgdg_b200: ext_noise must match images in shape and device, dtype %s" % want)
    return n


class PackedLut:
    """A 3D LUT in the library's device layout (vrgdg_lut3d_pack): `data` float32 [S^3 * 24] on a CUDA device."""

    def __init__(self, data, size):
        self.data, self.size = data, int(size)

    @property
    def device(self):
        return self.data.device


def pack_lut(lut, device=None):
    """[S,S,S,3] float32 table in the reference's [blue][green][red][rgb] order (CPU or CUDA) -> PackedLut."""
    if isinstance(lut, PackedLut):
        return lut
    if not isinstance(lut, torch.Tensor) or lut.ndim != 4 or lut.shape[3] != 3 or not (lut.shape[0] == lut.shape[1] == lut.shape[2]):
        raise ValueError("vrgdg_b200: lut must be float32 [S,S,S,3]")
    dev = torch.device(device) if device is not None else lut.device
    if dev.type != "cuda":
        raise RuntimeError("vrgdg_b200: LUTs are packed on a CUDA device; there is no CPU path")
    src = lut.to(device=dev, dtype=torch.float32).contiguous()
    S = int(src.shape[0])
    lib = nv.load_library()
    packed = torch.empty(int(lib.vrgdg_lut3d_packed_bytes(S)) // 4, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        nv.check(lib.vrgdg_lut3d_pack(nv.ptr(src), nv.ptr(packed), S, nv.stream_ptr(dev)))
    return PackedLut(packed, S)


def lut3d_apply(image, lut, dmin, dspan, blend=1.0, one_minus_blend=0.0):
    """VRGDG_LUTS._apply_cube_lut + strength blend.  image [B,H,W,3|4] CUDA; lut: PackedLut (or a [S,S,S,3] fp32 tensor,
    packed on the fly); dmin / dspan: 3 python floats each (dspan already clamped to >= 1e-6 in the image dtype)."""
    t = nv.require_cuda(image, "image")
    if t.ndim != 4 or t.shape[-1] not in (3, 4):
        raise ValueError("VRGDG_LUTS expects IMAGE input shaped like [batch, height, width, channels].")
    lut = pack_lut(lut, t.device)
    if lut.device != t.device:
        raise ValueError("vrgdg_b200: lut and image are on different devices")
    out = torch.empty_like(t)
    c3 = ctypes.c_float * 3
    lib = nv.load_library()
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_lut3d_apply(nv.ptr(t), nv.ptr(out), t.numel() // t.shape[-1], int(t.shape[-1]), nv.DTYPE_CODE[t.dtype],
                                       nv.ptr(lut.data), lut.size, c3(*[float(x) for x in dmin]), c3(*[float(x) for x in dspan]),
                                       _f32(blend), _f32(one_minus_blend), nv.stream_ptr(t.device)))
    return out


def grain(images, intensity, sat, one_minus_sat, seed, frame0=0, seed_mode=nv.SEED_PER_CLIP, ext_noise=None):
    t = _frames(images)
    n = None
    if ext_noise is not None:
        n = _noise(ext_noise, t)
    out = torch.empty_like(t)
    B, H, W, _ = t.shape
    lib = nv.load_library()
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_grain(nv.ptr(t), nv.ptr(out), B, H, W, nv.DTYPE_CODE[t.dtype], _f32(intensity), _f32(sat), _f32(one_minus_sat),
                                 ctypes.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), ctypes.c_int64(int(frame0)), int(seed_mode), nv.ptr(n),
                                 nv.stream_ptr(t.device)))
    return out


def grain_torch_global(images, intensity, sat, one_minus_sat, seed, philox_offset, frame0, clip_frames, draw_frames):
    """Frames [frame0, frame0 + B) of a clip of clip_frames frames with FastFilmGrain's grain drawn from a CUDA generator of seed `seed`
    at Philox offset `philox_offset`, one draw per `draw_frames` frames of the clip (vrgdg_grain_torch_global).  The generator is
    not advanced here."""
    t = _frames(images)
    out = torch.empty_like(t)
    B, H, W, _ = t.shape
    lib = nv.load_library()
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_grain_torch_global(nv.ptr(t), nv.ptr(out), B, H, W, nv.DTYPE_CODE[t.dtype], _f32(intensity), _f32(sat),
                                              _f32(one_minus_sat), ctypes.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF),
                                              ctypes.c_uint64(int(philox_offset) & 0xFFFFFFFFFFFFFFFF), ctypes.c_int64(int(frame0)),
                                              ctypes.c_int64(int(clip_frames)), ctypes.c_int64(int(draw_frames)), nv.stream_ptr(t.device)))
    return out


def grain_noise_torch_global(frames, seed, philox_offset, frame0, clip_frames, draw_frames):
    """The N(0,1) tensor grain_torch_global draws for `frames` (frames [frame0, frame0 + B) of the clip), shaped like `frames` and in
    their dtype: frame f's slice of the reference's torch.randn_like draw (vrgdg_grain_noise_torch_global).  It feeds the chain's
    ext_noise.  The generator is not advanced here."""
    t = _frames(frames)
    out = torch.empty_like(t)
    B, H, W, _ = t.shape
    lib = nv.load_library()
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_grain_noise_torch_global(nv.ptr(out), B, H, W, nv.DTYPE_CODE[t.dtype], ctypes.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF),
                                                    ctypes.c_uint64(int(philox_offset) & 0xFFFFFFFFFFFFFFFF), ctypes.c_int64(int(frame0)),
                                                    ctypes.c_int64(int(clip_frames)), ctypes.c_int64(int(draw_frames)), nv.stream_ptr(t.device)))
    return out


def torch_randn_increment(numel, device):
    """The Philox offset torch.randn of `numel` elements consumes on `device`'s CUDA generator (vrgdg_torch_randn_increment)."""
    inc = ctypes.c_int64(0)
    with torch.cuda.device(device):
        nv.check(nv.load_library().vrgdg_torch_randn_increment(ctypes.c_int64(int(numel)), ctypes.byref(inc)))
    return int(inc.value)


def grain_noise(B, H, W, seed, frame0=0, seed_mode=nv.SEED_PER_CLIP, device="cuda"):
    out = torch.empty((B, H, W, 3), dtype=torch.float32, device=device)
    lib = nv.load_library()
    with torch.cuda.device(out.device):
        nv.check(lib.vrgdg_grain_noise(nv.ptr(out), B, H, W, ctypes.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), ctypes.c_int64(int(frame0)),
                                       int(seed_mode), nv.stream_ptr(out.device)))
    return out


def stencil3x3(images, op, strength, border=nv.BORDER_REPLICATE):
    """3x3 sharpener on [B,H,W,3|4] CUDA frames (vrgdg_stencil3x3_ch).  RGBA frames are filtered on every channel, alpha included, as
    the reference's NumPy paths do; the torch-path ops (STENCIL_LAPLACIAN_GPU / STENCIL_SOBEL_GPU) and uint8 frames take 3 channels."""
    t = nv.require_cuda(images, "images")
    if t.ndim != 4 or t.shape[-1] not in (3, 4):
        raise ValueError("vrgdg_b200: images must be shaped [batch, height, width, 3 or 4], got %s" % (tuple(t.shape),))
    out = torch.empty_like(t)
    B, H, W, C = t.shape
    lib = nv.load_library()
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_stencil3x3_ch(nv.ptr(t), nv.ptr(out), B, H, W, C, nv.DTYPE_CODE[t.dtype], int(op), _f32(strength), int(border),
                                         nv.stream_ptr(t.device)))
    return out


def lab_moments(images, row0=0, rows=None):
    """Raw LAB sums per frame over rows [row0,row0+rows): float64 [B,7] = {n, S_L,S_a,S_b, S_LL,S_aa,S_bb}."""
    t = _frames(images)
    B, H, W, _ = t.shape
    rows = H - row0 if rows is None else rows
    lib = nv.load_library()
    sums = torch.empty((B, 7), dtype=torch.float64, device=t.device)
    nbytes = int(lib.vrgdg_lab_moments_scratch_bytes(B))
    scratch = torch.empty((max(nbytes, 8) // 8,), dtype=torch.float64, device=t.device)
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_lab_moments(nv.ptr(t), B, H, W, nv.DTYPE_CODE[t.dtype], int(row0), int(rows), nv.ptr(sums), nv.ptr(scratch),
                                       ctypes.c_int64(nbytes), nv.stream_ptr(t.device)))
    return sums


def colormatch_params(frame_sums, ref_sums):
    """[B,7] + [1|B,7] float64 CUDA -> [B,12] float32 {mu_img, sd_ref/sd_img, mu_ref, sd_img}."""
    fs = frame_sums.contiguous()
    rs = ref_sums.to(fs.device).contiguous()
    if fs.dtype != torch.float64 or rs.dtype != torch.float64 or fs.ndim != 2 or fs.shape[1] != 7 or rs.ndim != 2 or rs.shape[1] != 7:
        raise ValueError("vrgdg_b200: moment sums must be float64 [n,7]")
    if fs.device.type != "cuda":
        raise RuntimeError("vrgdg_b200: moment sums must live on a CUDA device")
    B = fs.shape[0]
    params = torch.empty((B, 12), dtype=torch.float32, device=fs.device)
    lib = nv.load_library()
    with torch.cuda.device(fs.device):
        nv.check(lib.vrgdg_colormatch_params(nv.ptr(fs), B, nv.ptr(rs), int(rs.shape[0]), nv.ptr(params), nv.stream_ptr(fs.device)))
    return params


def colormatch_apply(images, params, t_strength, one_minus_t):
    t = _frames(images)
    B, H, W, _ = t.shape
    p = params.contiguous()
    if p.dtype != torch.float32 or p.shape != (B, 12) or p.device != t.device:
        raise ValueError("vrgdg_b200: params must be float32 [B,12] on the images' device")
    out = torch.empty_like(t)
    lib = nv.load_library()
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_colormatch_apply(nv.ptr(t), nv.ptr(out), B, H, W, nv.DTYPE_CODE[t.dtype], nv.ptr(p), _f32(t_strength), _f32(one_minus_t),
                                            nv.stream_ptr(t.device)))
    return out


def _check_out(out, t):
    """A caller-supplied result tensor goes to the kernels as a raw pointer: it must be exactly what the wrappers would allocate."""
    if not isinstance(out, torch.Tensor) or out.shape != t.shape or out.dtype != t.dtype or out.device != t.device or not out.is_contiguous():
        raise ValueError("vrgdg_b200: `out` must be a contiguous tensor matching images in shape %s, dtype %s and device %s"
                         % (tuple(t.shape), t.dtype, t.device))
    nbytes = t.numel() * t.element_size()
    if nbytes and out.data_ptr() < t.data_ptr() + nbytes and t.data_ptr() < out.data_ptr() + nbytes:
        raise ValueError("vrgdg_b200: `out` must not overlap images (tile kernels read neighbouring pixels)")
    return out


def chain_apply(images, desc, ext_noise=None, keepalive=(), out=None, fast_math=False):
    """Run the fused chain described by a ChainDesc.  `keepalive` holds tensors the descriptor points to.  images [B,H,W,3|4]: RGBA
    frames take the LUT and the NumPy-path stencils only (vrgdg_chain_apply_ch), and no external noise."""
    t = nv.require_cuda(images, "images")
    if t.ndim != 4 or t.shape[-1] not in (3, 4):
        raise ValueError("vrgdg_b200: images must be shaped [batch, height, width, 3 or 4], got %s" % (tuple(t.shape),))
    B, H, W, C = t.shape
    if C == 4 and ext_noise is not None:
        raise ValueError("vrgdg_b200: ext_noise feeds the grain stage, which takes 3-channel frames; got 4 channels")
    out = torch.empty_like(t) if out is None else _check_out(out, t)
    lib = nv.load_library()
    with torch.cuda.device(t.device):
        if C == 4:
            nv.check(lib.vrgdg_chain_apply_ch(nv.ptr(t), nv.ptr(out), B, H, W, 4, nv.DTYPE_CODE[t.dtype], ctypes.byref(desc),
                                              nv.stream_ptr(t.device)))
        elif ext_noise is not None:
            n = _noise(ext_noise, t)
            nv.check(lib.vrgdg_chain_apply_ext(nv.ptr(t), nv.ptr(out), B, H, W, nv.DTYPE_CODE[t.dtype], ctypes.byref(desc), nv.ptr(n),
                                               nv.CHAIN_FAST_MATH if fast_math else 0, nv.stream_ptr(t.device)))
        else:
            nv.check(lib.vrgdg_chain_apply(nv.ptr(t), nv.ptr(out), B, H, W, nv.DTYPE_CODE[t.dtype], ctypes.byref(desc), nv.stream_ptr(t.device)))
    del keepalive
    return out


def _cm_flags(fast_math=False, recompute=False, serial=False):
    return (nv.CHAIN_FAST_MATH if fast_math else 0) | (nv.CHAIN_CM_RECOMPUTE if recompute else 0) | (nv.CHAIN_CM_SERIAL if serial else 0)


def chain_cm_scratch(images, recompute=False, group_frames=0):
    """Device scratch for chain_cm_apply on frames like `images` (reusable across calls with the same shape)."""
    t = _frames(images)
    B, H, W, _ = t.shape
    flags = nv.CHAIN_CM_RECOMPUTE if recompute else 0
    nbytes = int(nv.load_library().vrgdg_chain_cm_scratch_bytes(B, H, W, nv.DTYPE_CODE[t.dtype], flags, int(group_frames)))
    return torch.empty((max(nbytes, 256),), dtype=torch.uint8, device=t.device)


def chain_cm_apply(images, desc, ref_sums, ext_noise=None, out=None, fast_math=False, recompute=False, group_frames=0, scratch=None,
                   serial=False):
    """A chain with colour match in ONE library call (vrgdg_chain_cm_apply): statistics, parameters and the fused apply, group by
    group.  desc.colormatch_enabled / cm_t / cm_one_minus_t must be set; ref_sums: [1|B,7] float64 from lab_moments."""
    t = _frames(images)
    B, H, W, _ = t.shape
    out = torch.empty_like(t) if out is None else _check_out(out, t)
    rs = ref_sums.to(device=t.device, dtype=torch.float64).reshape(-1, 7).contiguous()
    flags = _cm_flags(fast_math, recompute, serial)
    lib = nv.load_library()
    need = int(lib.vrgdg_chain_cm_scratch_bytes(B, H, W, nv.DTYPE_CODE[t.dtype], flags, int(group_frames)))
    if scratch is None or scratch.numel() * scratch.element_size() < need or scratch.device != t.device:
        scratch = torch.empty((max(need, 256),), dtype=torch.uint8, device=t.device)
    n = _noise(ext_noise, t) if ext_noise is not None else None
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_chain_cm_apply(nv.ptr(t), nv.ptr(out), B, H, W, nv.DTYPE_CODE[t.dtype], ctypes.byref(desc), nv.ptr(rs), int(rs.shape[0]),
                                          nv.ptr(n), flags, nv.ptr(scratch), ctypes.c_int64(scratch.numel() * scratch.element_size()), int(group_frames),
                                          nv.stream_ptr(t.device)))
    return out, scratch


def chain_cm_apply_refs(images, desc, ref_frames, ext_noise=None, out=None, fast_math=False, recompute=False, group_frames=0, scratch=None,
                        serial=False):
    """chain_cm_apply against a reference clip in ONE library call (vrgdg_chain_cm_apply_refs): frame b is matched to ref_frames[b],
    whose statistics the call makes group by group.  ref_frames: [B,Hr,Wr,3] in the images' dtype on their device, any Hr x Wr.
    Bit-identical to chain_cm_apply(images, desc, lab_moments(ref_frames)).  Returns (out, scratch) as chain_cm_apply does."""
    t = _frames(images)
    r = _frames(ref_frames, "ref_frames")
    B, H, W, _ = t.shape
    if r.shape[0] != B or r.dtype != t.dtype or r.device != t.device:
        raise ValueError("vrgdg_b200: ref_frames must hold %d frames of dtype %s on %s, got %d of %s on %s"
                         % (B, t.dtype, t.device, r.shape[0], r.dtype, r.device))
    out = torch.empty_like(t) if out is None else _check_out(out, t)
    flags = _cm_flags(fast_math, recompute, serial)
    lib = nv.load_library()
    need = int(lib.vrgdg_chain_cm_scratch_bytes(B, H, W, nv.DTYPE_CODE[t.dtype], flags, int(group_frames)))
    if scratch is None or scratch.numel() * scratch.element_size() < need or scratch.device != t.device:
        scratch = torch.empty((max(need, 256),), dtype=torch.uint8, device=t.device)
    ref_sums = torch.empty((B, 7), dtype=torch.float64, device=t.device)
    n = _noise(ext_noise, t) if ext_noise is not None else None
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_chain_cm_apply_refs(nv.ptr(t), nv.ptr(out), B, H, W, nv.DTYPE_CODE[t.dtype], ctypes.byref(desc), nv.ptr(r),
                                               int(r.shape[1]), int(r.shape[2]), nv.ptr(ref_sums), nv.ptr(n), flags, nv.ptr(scratch),
                                               ctypes.c_int64(scratch.numel() * scratch.element_size()), int(group_frames),
                                               nv.stream_ptr(t.device)))
    return out, scratch


def chain_lab_moments(images, desc, ext_noise=None):
    """LAB sums [B,7] of stage 1 (grain) of `desc` applied to images; ext_noise: the N(0,1) tensor a chain_apply(ext_noise=...) will use."""
    t = _frames(images)
    B, H, W, _ = t.shape
    lib = nv.load_library()
    sums = torch.empty((B, 7), dtype=torch.float64, device=t.device)
    nbytes = int(lib.vrgdg_lab_moments_scratch_bytes(B))
    scratch = torch.empty((max(nbytes, 8) // 8,), dtype=torch.float64, device=t.device)
    n = _noise(ext_noise, t) if ext_noise is not None else None
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_chain_lab_moments_ext(nv.ptr(t), B, H, W, nv.DTYPE_CODE[t.dtype], ctypes.byref(desc), nv.ptr(n), nv.ptr(sums),
                                                 nv.ptr(scratch), ctypes.c_int64(nbytes), nv.stream_ptr(t.device)))
    return sums


def adjust(images, desc):
    """_apply_adjust_tensor with a prepared AdjustDesc (video_tools._adjust_desc builds it from a settings dict)."""
    t = _frames(images)
    B, H, W, _ = t.shape
    out = torch.empty_like(t)
    lib = nv.load_library()
    xx = yy = None
    if desc.enabled and desc.vignette_on:
        xx = torch.linspace(-1.0, 1.0, W, dtype=torch.float32).to(t.device)     # the reference's own ramps (:384-385)
        yy = torch.linspace(-1.0, 1.0, H, dtype=torch.float32).to(t.device)
    nbytes = int(lib.vrgdg_adjust_scratch_bytes(B, H, W, ctypes.byref(desc)))
    scratch = torch.empty((nbytes // 4,), dtype=torch.float32, device=t.device) if nbytes else None
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_adjust(nv.ptr(t), nv.ptr(out), B, H, W, nv.DTYPE_CODE[t.dtype], ctypes.byref(desc), nv.ptr(xx), nv.ptr(yy),
                                  nv.ptr(scratch), ctypes.c_int64(nbytes), nv.stream_ptr(t.device)))
    return out


RESIZE_MODES = {"nearest": 0, "bilinear": 1, "bicubic": 2, "area": 3}


def resize(images, out_h, out_w, mode, roi=None, resampled=None, offset=(0, 0)):
    """Resample roi=(x0, y0, w, h) of images [B,H,W,3|4] to resampled=(w, h) and place it at offset=(x, y) inside a zero-filled,
    clamped [B,out_h,out_w,3] result (vrgdg_resize; F.interpolate(..., align_corners=False) semantics)."""
    t = nv.require_cuda(images, "images")
    if t.ndim != 4 or t.shape[-1] not in (3, 4):
        raise ValueError("vrgdg_b200: expected frames [B,H,W,3|4], got %s" % (tuple(t.shape),))
    if t.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise ValueError("vrgdg_b200: resize needs float frames, got %s" % t.dtype)
    t = t.contiguous()
    B, H, W, C = t.shape
    x0, y0, sw, sh = roi if roi is not None else (0, 0, W, H)
    rw, rh = resampled if resampled is not None else (out_w, out_h)
    d = nv.ResizeDesc(RESIZE_MODES[mode], int(x0), int(y0), int(sw), int(sh), int(rw), int(rh), int(offset[0]), int(offset[1]))
    out = torch.empty((B, int(out_h), int(out_w), 3), dtype=t.dtype, device=t.device)
    lib = nv.load_library()
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_resize(nv.ptr(t), nv.ptr(out), B, H, W, C, int(out_h), int(out_w), nv.DTYPE_CODE[t.dtype], ctypes.byref(d),
                                  nv.stream_ptr(t.device)))
    return out


def blend(a, b, weight_a, weight_b):
    """clamp(a * weight_a + b * weight_b, 0, 1) (vrgdg_blend)."""
    ta, tb = nv.require_cuda(a, "a").contiguous(), nv.require_cuda(b, "b").contiguous()
    if ta.shape != tb.shape or ta.dtype != tb.dtype or ta.device != tb.device:
        raise ValueError("vrgdg_b200: blend operands differ (%s %s vs %s %s)" % (tuple(ta.shape), ta.dtype, tuple(tb.shape), tb.dtype))
    if ta.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise ValueError("vrgdg_b200: blend needs float frames, got %s" % ta.dtype)
    out = torch.empty_like(ta)
    lib = nv.load_library()
    with torch.cuda.device(ta.device):
        nv.check(lib.vrgdg_blend(nv.ptr(ta), nv.ptr(tb), nv.ptr(out), ta.numel(), nv.DTYPE_CODE[ta.dtype], float(weight_a), float(weight_b),
                                 nv.stream_ptr(ta.device)))
    return out


def restore_blend(enhanced, originals, mode, weight_orig, weight_restored, roi=None, n_restored=None):
    """The restore node in one launch (vrgdg_restore_blend): roi=(x0, y0, w, h) of enhanced [Be,He,We,3|4] is resampled to the
    originals' size, and for the first n_restored frames (default min(B, Be)) clamp(originals * weight_orig + restored * weight_restored,
    0, 1) replaces their RGB; the rest of originals [B,H,W,3|4] (alpha, later frames) is clamped.  Equals resize -> blend -> clamp."""
    te, to = nv.require_cuda(enhanced, "enhanced"), nv.require_cuda(originals, "originals")
    if te.ndim != 4 or te.shape[-1] not in (3, 4) or to.ndim != 4 or to.shape[-1] not in (3, 4):
        raise ValueError("vrgdg_b200: restore_blend expects frames [B,H,W,3|4], got %s and %s" % (tuple(te.shape), tuple(to.shape)))
    if te.dtype != to.dtype or te.device != to.device:
        raise ValueError("vrgdg_b200: restore_blend operands differ (%s on %s vs %s on %s)" % (te.dtype, te.device, to.dtype, to.device))
    if to.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise ValueError("vrgdg_b200: restore_blend needs float frames, got %s" % to.dtype)
    Be, He, We, Ce = te.shape
    B, H, W, Co = to.shape
    n = min(B, Be) if n_restored is None else int(n_restored)
    if not 0 <= n <= min(B, Be):
        raise ValueError("vrgdg_b200: n_restored %d outside [0, %d]" % (n, min(B, Be)))
    x0, y0, sw, sh = roi if roi is not None else (0, 0, We, He)
    d = nv.ResizeDesc(RESIZE_MODES[mode], int(x0), int(y0), int(sw), int(sh), int(W), int(H), 0, 0)
    out = torch.empty_like(to)
    lib = nv.load_library()
    with torch.cuda.device(to.device):
        nv.check(lib.vrgdg_restore_blend(nv.ptr(te), nv.ptr(to), nv.ptr(out), B, n, He, We, Ce, H, W, Co, nv.DTYPE_CODE[to.dtype],
                                         ctypes.byref(d), float(weight_orig), float(weight_restored), nv.stream_ptr(to.device)))
    return out


def hist_counts(images, row0=0, rows=None):
    """Per-frame, per-channel (R, G, B) 256-bin counts over rows [row0,row0+rows): int32 [B,3,256] (histogram colour match, a labelled
    extension: vrgdg_hist_counts).  Counts are exact, so row-sharded counts of one image add up to the whole image's."""
    t = _frames(images)
    B, H, W, _ = t.shape
    rows = H - row0 if rows is None else rows
    counts = torch.empty((B, 3, 256), dtype=torch.int32, device=t.device)
    lib = nv.load_library()
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_hist_counts(nv.ptr(t), B, H, W, nv.DTYPE_CODE[t.dtype], int(row0), int(rows), nv.ptr(counts), nv.stream_ptr(t.device)))
    return counts


def histmatch_tables(frame_counts, ref_counts):
    """[B,3,256] + [1|B,3,256] int32 counts -> [B,3,256,2] float32 {T[k], T[k+1]-T[k]}: the monotone map ref_CDF^-1(frame_CDF)."""
    fc = frame_counts.contiguous()
    rc = ref_counts.to(fc.device).contiguous()
    if fc.dtype != torch.int32 or rc.dtype != torch.int32 or fc.ndim != 3 or fc.shape[1:] != (3, 256) or rc.ndim != 3 or rc.shape[1:] != (3, 256):
        raise ValueError("vrgdg_b200: histogram counts must be int32 [n,3,256]")
    if fc.device.type != "cuda":
        raise RuntimeError("vrgdg_b200: histogram counts must live on a CUDA device")
    B = int(fc.shape[0])
    tables = torch.empty((B, 3, 256, 2), dtype=torch.float32, device=fc.device)
    lib = nv.load_library()
    with torch.cuda.device(fc.device):
        nv.check(lib.vrgdg_histmatch_tables(nv.ptr(fc), B, nv.ptr(rc), int(rc.shape[0]), nv.ptr(tables), nv.stream_ptr(fc.device)))
    return tables


def histmatch_apply(images, tables, t_strength, one_minus_t):
    t = _frames(images)
    B, H, W, _ = t.shape
    tb = tables.contiguous()
    if tb.dtype != torch.float32 or tuple(tb.shape) != (B, 3, 256, 2) or tb.device != t.device:
        raise ValueError("vrgdg_b200: tables must be float32 [B,3,256,2] on the images' device")
    out = torch.empty_like(t)
    lib = nv.load_library()
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_histmatch_apply(nv.ptr(t), nv.ptr(out), B, H, W, nv.DTYPE_CODE[t.dtype], nv.ptr(tb), _f32(t_strength), _f32(one_minus_t),
                                           nv.stream_ptr(t.device)))
    return out


def histmatch_apply_refs(images, ref_frames, t_strength, one_minus_t, scratch=None):
    """Histogram colour match against a reference clip in ONE library call (vrgdg_histmatch_apply_refs): frame b is matched to
    ref_frames[b].  ref_frames: [B,Hr,Wr,3] in the images' dtype on their device, any Hr x Wr.  torch.equal to
    histmatch_apply(images, histmatch_tables(hist_counts(images), hist_counts(ref_frames)), t_strength, one_minus_t).
    Returns (out, scratch); hand the scratch back to the next call to reuse it."""
    t = _frames(images)
    r = _frames(ref_frames, "ref_frames")
    B, H, W, _ = t.shape
    if r.shape[0] != B or r.dtype != t.dtype or r.device != t.device:
        raise ValueError("vrgdg_b200: ref_frames must hold %d frames of dtype %s on %s, got %d of %s on %s"
                         % (B, t.dtype, t.device, r.shape[0], r.dtype, r.device))
    out = torch.empty_like(t)
    lib = nv.load_library()
    need = int(lib.vrgdg_histmatch_refs_scratch_bytes(B))
    if scratch is None or scratch.numel() * scratch.element_size() < need or scratch.device != t.device:
        scratch = torch.empty((max(need, 256),), dtype=torch.uint8, device=t.device)
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_histmatch_apply_refs(nv.ptr(t), nv.ptr(out), B, H, W, nv.DTYPE_CODE[t.dtype], nv.ptr(r), int(r.shape[1]),
                                                int(r.shape[2]), _f32(t_strength), _f32(one_minus_t), nv.ptr(scratch),
                                                ctypes.c_int64(scratch.numel() * scratch.element_size()), nv.stream_ptr(t.device)))
    return out, scratch


def temporal_sharpen(images, strength, prev_frame=None, next_frame=None):
    """3-frame temporal unsharp over a clip [T,H,W,3] (configs[4]; labelled extension, see vrgdg_temporal_sharpen).  prev_frame /
    next_frame: [H,W,3] (or [1,H,W,3]) neighbours of the first / last frame when the clip is a shard of a longer one."""
    t = _frames(images)
    B, H, W, _ = t.shape

    def halo(h, name):
        if h is None:
            return None
        h = nv.require_cuda(h, name)
        if h.numel() != H * W * 3 or h.dtype != t.dtype or h.device != t.device:
            raise ValueError("vrgdg_b200: %s must be one frame [%d,%d,3] of dtype %s on %s" % (name, H, W, t.dtype, t.device))
        return h
    p, n = halo(prev_frame, "prev_frame"), halo(next_frame, "next_frame")
    out = torch.empty_like(t)
    lib = nv.load_library()
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_temporal_sharpen(nv.ptr(t), nv.ptr(out), B, H, W, nv.DTYPE_CODE[t.dtype], _f32(strength), nv.ptr(p), nv.ptr(n),
                                            nv.stream_ptr(t.device)))
    return out


_LANCZOS_TABLES = {}


def lanczos4_tables(src_size, dst_size, device):
    """(ofs int32 [dst], coef int16 [dst,8]) of one axis on `device`; built on the host by the library (OpenCV's recipe), cached."""
    key = (int(src_size), int(dst_size), str(device))
    hit = _LANCZOS_TABLES.get(key)
    if hit is None:
        ofs = np.empty(int(dst_size), dtype=np.int32)
        coef = np.empty((int(dst_size), 8), dtype=np.int16)
        lib = nv.load_library()
        nv.check(lib.vrgdg_lanczos4_tables(int(src_size), int(dst_size), ofs.ctypes.data_as(ctypes.c_void_p), coef.ctypes.data_as(ctypes.c_void_p)))
        if len(_LANCZOS_TABLES) > 64:
            _LANCZOS_TABLES.clear()
        hit = _LANCZOS_TABLES[key] = (torch.from_numpy(ofs).to(device), torch.from_numpy(coef).to(device))
    return hit


def resize_lanczos4_u8(frames_u8, out_h, out_w, max_scratch_bytes=1 << 30):
    """cv2.resize(INTER_LANCZOS4) of uint8 CUDA frames [B,H,W,3] -> [B,out_h,out_w,3], bit-identical to OpenCV
    (vrgdg_lanczos4_resize_u8).  Frames are processed in groups so that the int32 scratch stays below max_scratch_bytes."""
    if not isinstance(frames_u8, torch.Tensor) or frames_u8.device.type != "cuda" or frames_u8.dtype != torch.uint8 or frames_u8.ndim != 4 \
            or frames_u8.shape[-1] != 3:
        raise ValueError("vrgdg_b200: expected a CUDA uint8 tensor [B,H,W,3]")
    s = frames_u8.contiguous()
    B, H, W, _ = s.shape
    oh, ow = max(1, int(out_h)), max(1, int(out_w))
    out = torch.empty((B, oh, ow, 3), dtype=torch.uint8, device=s.device)
    if B == 0:
        return out
    if H < 1 or W < 1:
        raise ValueError("vrgdg_b200: cannot resize empty frames")
    lib = nv.load_library()
    xo, xc = lanczos4_tables(W, ow, s.device)
    yo, yc = lanczos4_tables(H, oh, s.device)
    per_frame = int(lib.vrgdg_lanczos4_scratch_bytes(1, H, ow))
    group = max(1, min(B, max_scratch_bytes // max(1, per_frame)))
    scratch = torch.empty((group * per_frame // 4,), dtype=torch.int32, device=s.device)
    with torch.cuda.device(s.device):
        for b0 in range(0, B, group):
            n = min(group, B - b0)
            nv.check(lib.vrgdg_lanczos4_resize_u8(nv.ptr(s[b0:b0 + n]), nv.ptr(out[b0:b0 + n]), n, H, W, oh, ow, nv.ptr(xo), nv.ptr(xc), nv.ptr(yo),
                                                  nv.ptr(yc), nv.ptr(scratch), ctypes.c_int64(n * per_frame), nv.stream_ptr(s.device)))
    return out


def u8bgr_to_rgb(frames_u8, dtype=torch.float32):
    """uint8 BGR [..., 3] CUDA -> RGB float (x/255)."""
    if frames_u8.device.type != "cuda" or frames_u8.dtype != torch.uint8 or frames_u8.shape[-1] != 3:
        raise ValueError("vrgdg_b200: expected a CUDA uint8 tensor [...,3]")
    s = frames_u8.contiguous()
    out = torch.empty(s.shape, dtype=dtype, device=s.device)
    lib = nv.load_library()
    with torch.cuda.device(s.device):
        nv.check(lib.vrgdg_u8bgr_to_rgb(nv.ptr(s), nv.ptr(out), s.numel() // 3, nv.DTYPE_CODE[dtype], nv.stream_ptr(s.device)))
    return out


def rgb_to_u8bgr(frames):
    t = nv.require_cuda(frames, "frames")
    if t.shape[-1] != 3:
        raise ValueError("vrgdg_b200: expected [...,3]")
    out = torch.empty(t.shape, dtype=torch.uint8, device=t.device)
    lib = nv.load_library()
    with torch.cuda.device(t.device):
        nv.check(lib.vrgdg_rgb_to_u8bgr(nv.ptr(t), nv.ptr(out), t.numel() // 3, nv.DTYPE_CODE[t.dtype], nv.stream_ptr(t.device)))
    return out

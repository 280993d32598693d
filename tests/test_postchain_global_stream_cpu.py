"""VRGDG_B200_PostChain's grain from the global CUDA generator (VRGDG_GRAIN_NOISE=torch_cuda) without a GPU: the noise kernel's
work-item -> element mapping compiled for the host (tests/hostcheck/global_noise.cpp) against torch_randn_site, the new C entry
point's refusals, which return before any CUDA call, and the node's refusals and default path."""
import ctypes
import importlib
import os
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostcheck", "global_noise.cpp")
u32p = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")
MAX_THREADS_PER_SM = 2048


@pytest.fixture(scope="module")
def gn(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("global_noise") / "libglobal_noise.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", so], check=True)
    lib = ctypes.CDLL(so)
    lib.gn_walk.restype = ctypes.c_uint32
    lib.gn_walk.argtypes = [ctypes.c_uint32] * 8 + [u32p, u32p, u32p]
    lib.gn_sites.argtypes = [u32p, u32p, ctypes.c_uint64, u32p]
    lib.gn_threads.restype = ctypes.c_uint32
    lib.gn_threads.argtypes = [ctypes.c_uint64, ctypes.c_int, ctypes.c_int]
    return lib


def walk(gn, frame0, frames, n, step, clip, sms):
    T_full = gn.gn_threads(step * n, sms, MAX_THREADS_PER_SM)
    last = (clip - 1) // step
    T_last = gn.gn_threads((min(clip, (last + 1) * step) - last * step) * n, sms, MAX_THREADS_PER_SM)
    size = frames * n
    visits = np.zeros(size, dtype=np.uint32)
    site = np.zeros(3 * size, dtype=np.uint32)
    draw = np.zeros(size, dtype=np.uint32)
    rows = gn.gn_walk(frame0, frames, n, step, clip, T_full, T_last, 1 << 20, visits, site, draw)
    assert rows > 0
    return visits, site.reshape(size, 3), draw, T_full, T_last, rows


# (H, W, clip frames, draw frames, windows as (frame0, frames)): partial last draws, windows that start and end mid-draw, one window
# per draw and one over the whole clip; 17x23 and 270x480 frames put several frames in one row of 4T elements, 1080p several rows
# in one frame
CASES = [
    ((17, 23), 7, 3, [(0, 7), (1, 2), (2, 3), (5, 2), (6, 1), (3, 4)]),
    ((17, 23), 7, 4, [(0, 7), (3, 2), (4, 3), (1, 6)]),
    ((17, 23), 7, 1, [(0, 7), (2, 3)]),
    ((17, 23), 7, 7, [(0, 7), (2, 3), (6, 1)]),
    ((270, 480), 7, 3, [(0, 7), (1, 3), (5, 2), (2, 1)]),
    ((270, 480), 5, 4, [(3, 2), (0, 5), (4, 1)]),
    ((1080, 1920), 5, 2, [(1, 1), (4, 1), (2, 1)]),
]


@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("shape,clip,step,windows", CASES, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else None)
def test_work_items_store_every_window_element_once_at_its_aten_site(gn, sms, shape, clip, step, windows):
    n = shape[0] * shape[1] * 3
    for frame0, frames in windows:
        visits, site, draw, T_full, T_last, rows = walk(gn, frame0, frames, n, step, clip, sms)
        assert visits.min() == 1 and visits.max() == 1, (frame0, frames)
        e = np.arange(frames * n, dtype=np.int64)
        f = frame0 + e // n                                   # absolute frame of each window element
        j = f // step
        li = ((f - j * step) * n + e % n).astype(np.uint32)   # its index in draw j
        T = np.where((j + 1) * step >= clip, T_last, T_full).astype(np.uint32)
        assert np.array_equal(draw, j.astype(np.uint32))
        want = np.zeros((frames * n, 3), dtype=np.uint32)
        gn.gn_sites(li, T, frames * n, want.reshape(-1))
        assert np.array_equal(site, want), (frame0, frames)
        # the rows are those of the window alone: at most one partly used row at each end of each draw it touches
        draws = int(j[-1] - j[0] + 1)
        assert rows <= draws * ((step * n - 1) // (4 * T_full) + 1)
        assert rows <= (frames * n) // (4 * T_last) + 2 * draws


def _lib(pkg):
    nv = pkg._native
    return nv, nv.load_library()


def test_noise_entry_point_is_declared_and_typed(pkg):
    nv, lib = _lib(pkg)
    hdr = open(os.path.join(ROOT, "include", "vrgdg_b200.h")).read()
    assert "VRGDG_API int vrgdg_grain_noise_torch_global(void* noise, int B, int H, int W, int dtype, uint64_t seed, " \
           "uint64_t philox_offset," in hdr
    restype, argtypes = nv.SIGNATURES["vrgdg_grain_noise_torch_global"]
    assert restype is ctypes.c_int and len(argtypes) == 11
    assert lib.vrgdg_grain_noise_torch_global is not None


def test_noise_entry_point_refuses_what_the_grain_entry_point_refuses(pkg):
    """the same refusals with the same messages as vrgdg_grain_torch_global, before any CUDA call"""
    nv, lib = _lib(pkg)
    src, dst = ctypes.c_void_p(256), ctypes.c_void_p(512)          # non-null, aligned, never dereferenced

    def call(which, B, H, W, dtype, offset=0, frame0=0, clip=None, draw=4):
        tail = (ctypes.c_uint64(42), ctypes.c_uint64(offset), ctypes.c_int64(frame0), ctypes.c_int64(B if clip is None else clip),
                ctypes.c_int64(draw), None)
        if which == "grain":
            rc = lib.vrgdg_grain_torch_global(src, dst, B, H, W, dtype, ctypes.c_float(0.04), ctypes.c_float(0.5), ctypes.c_float(0.5), *tail)
        else:
            rc = lib.vrgdg_grain_noise_torch_global(dst, B, H, W, dtype, *tail)
        return rc, lib.vrgdg_last_error().decode()

    cases = [
        (dict(B=2, H=8, W=8, dtype=nv.U8BGR), nv.E_UNSUPPORTED, "float frames"),
        (dict(B=2, H=8, W=8, dtype=7), nv.E_INVALID, "unknown dtype"),
        (dict(B=2, H=8, W=8, dtype=nv.F32, offset=6), nv.E_INVALID, "multiple of 4"),
        (dict(B=2, H=8, W=8, dtype=nv.F32, draw=0), nv.E_INVALID, "draw_frames"),
        (dict(B=2, H=8, W=8, dtype=nv.F32, frame0=-1, clip=4), nv.E_INVALID, "clip of 4 frames"),
        (dict(B=2, H=8, W=8, dtype=nv.F32, frame0=3, clip=4), nv.E_INVALID, "clip of 4 frames"),
        (dict(B=2, H=8, W=8, dtype=nv.F32, clip=2**31), nv.E_INVALID, "clip of"),
        (dict(B=22, H=2160, W=3840, dtype=nv.F32, draw=22), nv.E_UNSUPPORTED, "exceeds 32-bit indexing"),
        (dict(B=1, H=2160, W=3840, dtype=nv.F32, clip=30, draw=0x7FFFFFFF), nv.E_UNSUPPORTED, "exceeds 32-bit indexing"),
        (dict(B=44, H=2160, W=3840, dtype=nv.BF16, draw=44), nv.E_UNSUPPORTED, "exceeds 32-bit indexing"),
        (dict(B=1, H=16384, W=16384, dtype=nv.F32, draw=1), nv.E_UNSUPPORTED, "exceeds 32-bit indexing"),
        (dict(B=2, H=-1, W=8, dtype=nv.F32), nv.E_INVALID, "negative shape"),
    ]
    for kw, code, text in cases:
        rc_g, msg_g = call("grain", **kw)
        rc_n, msg_n = call("noise", **kw)
        assert rc_g == rc_n == code, (kw, rc_g, rc_n, msg_n)
        assert text in msg_n
        assert msg_n == msg_g.replace("vrgdg_grain_torch_global", "vrgdg_grain_noise_torch_global"), (msg_g, msg_n)
    # nothing to draw is a success before any CUDA call
    assert call("noise", 0, 2160, 3840, nv.F32, clip=0, draw=22)[0] == nv.VRGDG_OK
    assert call("noise", 3, 0, 3840, nv.F16, clip=3, draw=1)[0] == nv.VRGDG_OK
    # a null tensor with frames to draw
    assert lib.vrgdg_grain_noise_torch_global(None, 1, 8, 8, nv.F32, ctypes.c_uint64(1), ctypes.c_uint64(0), ctypes.c_int64(0),
                                              ctypes.c_int64(1), ctypes.c_int64(1), None) == nv.E_INVALID


def _node(pkg):
    return pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_PostChain"]()


def test_node_refusals_come_before_any_generator_or_device_work(pkg, monkeypatch):
    """under torch_cuda a draw past 32-bit indexing, and any unknown VRGDG_GRAIN_NOISE value, raise ValueError before the CPU generator
    is drawn from and before the compute device is looked up (which would raise RuntimeError without a GPU)"""
    node = _node(pkg)
    state = torch.get_rng_state()
    x = torch.zeros(1, 4, 4, 3)
    for raw in ("mt19937", "torch"):
        monkeypatch.setenv("VRGDG_GRAIN_NOISE", raw)
        with pytest.raises(ValueError, match="VRGDG_GRAIN_NOISE=%s" % raw):
            node.apply_chain(x, 0.04, 0.5, 1.0, "none", 10.0, "unsharp", 0.5, False, 8)
    monkeypatch.setenv("VRGDG_GRAIN_NOISE", "torch_cuda")
    clip = torch.zeros(1, 1, 1, 3).expand(30, 2160, 3840, 3)      # 30 x 4K fp32 frames without the memory
    for batch_size in (0, 22, 500):
        with pytest.raises(ValueError, match="VRGDG_B200_PostChain with VRGDG_GRAIN_NOISE=torch_cuda.*batch_size=%d" % batch_size):
            node.apply_chain(clip, 0.04, 0.5, 1.0, "none", 10.0, "unsharp", 0.5, False, batch_size)
    with pytest.raises(ValueError, match="lower batch_size"):                 # 16-bit draws: 44 x 4K frames
        node.apply_chain(torch.zeros(1, 1, 1, 3, dtype=torch.float16).expand(44, 2160, 3840, 3), 0.04, 0.5, 1.0, "none", 10.0,
                         "none", 0.5, False, 0)
    # RGBA frames keep their own refusal, in either mode
    with pytest.raises(ValueError, match="grain_intensity must be 0 for RGBA"):
        node.apply_chain(torch.zeros(1, 4, 4, 4), 0.04, 0.5, 1.0, "none", 10.0, "unsharp", 0.5, False, 8)
    assert torch.equal(state, torch.get_rng_state())
    types = node.INPUT_TYPES()
    assert "VRGDG_GRAIN_NOISE=torch_cuda" in types["required"]["batch_size"][1]["tooltip"]


class _Recorder:
    """stands in for PostChain and the frame loop: records the chain's grain spec"""

    def __init__(self):
        self.grains = []

    def chain(self, grain=None, **kw):
        self.grains.append(grain)

        class C:
            device = torch.device("cpu")

            def make_fn(self):
                return None
        return C()


@pytest.mark.parametrize("raw", [None, "", "vrgdg", "torch_cuda"])
def test_node_default_path_and_zero_intensity_keep_the_cpu_generator_as_today(pkg, monkeypatch, raw):
    """unset / vrgdg: one draw_seed() from the CPU generator, as before; grain_intensity 0: no draw in any mode and no generator read"""
    cn = importlib.import_module(pkg.__name__ + ".chain_nodes")
    rec = _Recorder()
    monkeypatch.setattr(cn, "PostChain", rec.chain)
    monkeypatch.setattr(cn, "compute_device", lambda images=None: torch.device("cpu"))
    monkeypatch.setattr(cn, "run_frames", lambda images, *a: images.clone())
    monkeypatch.setattr(cn, "GlobalStreamDraws", None)          # any use of the global stream fails loudly
    if raw is None:
        monkeypatch.delenv("VRGDG_GRAIN_NOISE", raising=False)
    else:
        monkeypatch.setenv("VRGDG_GRAIN_NOISE", raw)
    node = _node(pkg)
    x = torch.rand(3, 8, 8, 3)
    # grain_intensity 0: nothing is drawn in any mode
    torch.manual_seed(11)
    state = torch.get_rng_state()
    node.apply_chain(x, 0.0, 0.5, 1.0, "none", 10.0, "unsharp", 0.5, False, 2)
    assert torch.equal(state, torch.get_rng_state()) and rec.grains == [None]
    if raw == "torch_cuda":
        return
    torch.manual_seed(11)
    want = int(torch.randint(0, 2**62, (1,), dtype=torch.int64).item())
    after = torch.get_rng_state()
    torch.manual_seed(11)
    node.apply_chain(x, 0.04, 0.5, 1.0, "none", 10.0, "unsharp", 0.5, False, 2)
    assert rec.grains[-1] == dict(intensity=0.04, saturation_mix=0.5, seed=want)
    assert torch.equal(after, torch.get_rng_state())


def test_chain_refuses_ext_noise_and_uint8_frames_with_the_global_stream(pkg):
    """a caller's ext_noise would replace the stream, and uint8 frames are no IMAGE tensors: both raise before any device work"""
    spec = dict(seed=1, philox_offset=0, clip_frames=2, draw_frames=1)
    chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, torch_global=spec), device="cuda:0")
    x = torch.zeros(2, 4, 4, 3)
    with pytest.raises(ValueError, match="ext_noise cannot replace it"):
        chain(x, ext_noise=torch.zeros_like(x))
    with pytest.raises(ValueError, match="got uint8"):
        chain(torch.zeros(2, 4, 4, 3, dtype=torch.uint8))
    with pytest.raises(ValueError, match="got uint8"):
        chain.run_host(torch.zeros(2, 4, 4, 3, dtype=torch.uint8))
    with pytest.raises(ValueError, match="takes 3-channel frames"):
        chain.run_host(torch.zeros(2, 4, 4, 4))

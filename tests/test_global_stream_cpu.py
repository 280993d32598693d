"""FastFilmGrain's global-generator stream (VRGDG_GRAIN_NOISE=torch_cuda) without a GPU: the draw geometry, the Philox offset and
the counter increment of csrc/vrgdg_math.cuh compiled for the host (tests/hostcheck/global_stream.cpp) against a restatement of
the reference's mini-batch loop, ATen's calc_execution_policy and curand's skipahead; the C ABI's refusals, which return before any
CUDA call; and the node's environment variable and argument checks."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostcheck", "global_stream.cpp")
u32p = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")
u64p = np.ctypeslib.ndpointer(dtype=np.uint64, flags="C_CONTIGUOUS")
MAX_THREADS_PER_SM = 2048


@pytest.fixture(scope="module")
def gs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("global_stream") / "libglobal_stream.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", so], check=True)
    lib = ctypes.CDLL(so)
    lib.gs_threads.restype = ctypes.c_uint32
    lib.gs_threads.argtypes = [ctypes.c_uint64, ctypes.c_int, ctypes.c_int]
    lib.gs_bits_fresh.argtypes = [ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, u32p]
    lib.gs_bits_at.argtypes = [ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64, u32p]
    lib.gs_philox.argtypes = [u32p, u32p, u32p]
    lib.gs_increment.restype = ctypes.c_uint64
    lib.gs_increment.argtypes = [ctypes.c_uint64, ctypes.c_uint32]
    lib.gs_global_draw.argtypes = [ctypes.c_uint32] * 6 + [ctypes.c_uint64, u64p]
    return lib


def aten_threads(numel, sms):
    """calc_execution_policy: 256-thread blocks, grid capped at SMs x (max threads per SM / 256)"""
    return 256 * min(sms * (MAX_THREADS_PER_SM // 256), (numel + 255) // 256)


def aten_increment(numel, sms):
    """calc_execution_policy's counter_offset (4 curand calls per unrolled iteration), rounded to a multiple of 4 by
    philox_cuda_state; an empty draw returns before it"""
    if numel == 0:
        return 0
    T = aten_threads(numel, sms)
    inc = ((numel - 1) // (T * 4) + 1) * 4
    return (inc + 3) // 4 * 4


def reference_draws(B, step, n, o0, sms):
    """FastFilmGrain's loop (nodes.py:46-62): one randn_like per mini-batch, each at the generator's offset before it.
    Returns [(first frame, frames, numel, T, offset)] and the offset after the call."""
    draws, o = [], o0
    for i in range(0, B, step):
        frames = min(step, B - i)
        numel = frames * n
        draws.append((i, frames, numel, aten_threads(numel, sms), o))
        o += aten_increment(numel, sms)
    return draws, o


def curand_counter(idx, offset, k):
    """curand_init(seed, idx, offset) then k curand4 calls: skipahead_sequence adds idx to the upper 64 counter bits, skipahead
    adds offset / 4 (offset % 4 == 0) and every curand4 one more, all as one 128-bit counter"""
    c = ((idx << 64) + offset // 4 + k) % (1 << 128)
    return [(c >> s) & 0xFFFFFFFF for s in (0, 32, 64, 96)]


@pytest.mark.parametrize("sms", [132, 114, 1])
def test_increment_is_atens_counter_offset(gs, sms):
    T_full = aten_threads(1 << 40, sms)
    for numel in (0, 1, 3, 255, 256, 257, 4 * T_full - 1, 4 * T_full, 4 * T_full + 1, 17 * 23 * 3, 1920 * 1080 * 3,
                  4 * 1920 * 1080 * 3, 3840 * 2160 * 3, 3 * 3840 * 2160 * 3):
        T = gs.gs_threads(max(numel, 1), sms, MAX_THREADS_PER_SM)
        assert gs.gs_increment(numel, T) == aten_increment(numel, sms), numel
    # H100 SXM: T = 270336, so a 1080p fp32 frame takes 4 * 6 and a 4K frame 4 * 24
    assert gs.gs_increment(1920 * 1080 * 3, 270336) == 24 and gs.gs_increment(3840 * 2160 * 3, 270336) == 96
    assert gs.gs_increment(17 * 23 * 3, 1280) == 4


def test_offset_counter_layout_and_carry(gs):
    """element li at Philox offset o reads Philox(counter of curand_init(seed, idx, o) after k calls); offset 0 is the fresh
    generator's stream, and k + o/4 carries into the second counter word"""
    T = 270336
    lis = (0, 1, T - 1, T, 3 * T + 5, 4 * T, 4 * T + 7, 9 * T + 11, 3840 * 2160 * 3 - 1)
    offsets = (0, 4, 96, 4 * (2**32 - 1), 4 * (2**32 - 5), 2**34, 2**34 + 12, 4 * (2**40 + 3), 2**64 - 4)
    for seed in (0, 67280421310721, 2**64 - 1):
        key = np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint32)
        for li in lis:
            k, r = divmod(li, 4 * T)
            idx = r % T
            fresh = np.zeros(4, dtype=np.uint32)
            gs.gs_bits_fresh(seed, li, T, fresh)
            for o in offsets:
                want = np.zeros(4, dtype=np.uint32)
                gs.gs_philox(np.array(curand_counter(idx, o, k), dtype=np.uint32), key, want)
                got = np.zeros(4, dtype=np.uint32)
                gs.gs_bits_at(seed, li, T, o, got)
                assert np.array_equal(got, want), (seed, li, o)
                if o == 0:
                    assert np.array_equal(got, fresh)
    # the carry itself: k = 1 at o/4 = 2^32 - 1 reads counter words {0, 1}
    assert curand_counter(5, 4 * (2**32 - 1), 1) == [0, 1, 5, 0]


@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("B,batch_size", [(7, 0), (7, 1), (7, 3), (7, 4), (7, 7), (7, 9), (1, 4), (16, 4)])
@pytest.mark.parametrize("shape", [(17, 23), (1080, 1920), (2160, 3840)], ids=lambda s: "%dx%d" % s)
def test_draw_geometry_is_the_reference_loop(gs, sms, B, batch_size, shape):
    """every frame's draw, element base, numel, T and offset, partial last draws included, and the offset after the call"""
    n = shape[0] * shape[1] * 3
    step = min(batch_size, B) if batch_size > 0 else B
    o0 = 4 * (2**32 - 5)
    draws, o_end = reference_draws(B, step, n, o0, sms)
    T_full = gs.gs_threads(step * n, sms, MAX_THREADS_PER_SM)
    last_numel = (B - (B - 1) // step * step) * n
    T_last = gs.gs_threads(last_numel, sms, MAX_THREADS_PER_SM)
    got = np.zeros(5, dtype=np.uint64)
    for j, (first, frames, numel, T, o) in enumerate(draws):
        for f in range(first, first + frames):
            gs.gs_global_draw(f, step, B, n, T_full, T_last, o0, got)
            assert got.tolist() == [j, (f - first) * n, numel, T, o], (f, got.tolist())
    # the node's total: full draws times the full increment, plus the remainder's
    total = (B // step) * aten_increment(step * n, sms) + aten_increment((B % step) * n, sms)
    assert o0 + total == o_end


def _lib(pkg):
    nv = pkg._native
    return nv, nv.load_library()


def test_abi_refusals_without_a_gpu(pkg):
    nv, lib = _lib(pkg)
    src, dst = ctypes.c_void_p(256), ctypes.c_void_p(512)          # non-null, aligned, never dereferenced

    def call(B, H, W, dtype, offset=0, frame0=0, clip=None, draw=4):
        return lib.vrgdg_grain_torch_global(src, dst, B, H, W, dtype, ctypes.c_float(0.04), ctypes.c_float(0.5), ctypes.c_float(0.5),
                                            ctypes.c_uint64(42), ctypes.c_uint64(offset), ctypes.c_int64(frame0),
                                            ctypes.c_int64(B if clip is None else clip), ctypes.c_int64(draw), None)

    def expect(rc, code, text):
        assert rc == code, (rc, lib.vrgdg_last_error())
        assert text in lib.vrgdg_last_error().decode()

    expect(call(2, 8, 8, nv.U8BGR), nv.E_UNSUPPORTED, "float frames")
    expect(call(2, 8, 8, 7), nv.E_INVALID, "unknown dtype")
    expect(call(2, 8, 8, nv.F32, offset=6), nv.E_INVALID, "multiple of 4")
    expect(call(2, 8, 8, nv.F32, draw=0), nv.E_INVALID, "draw_frames")
    expect(call(2, 8, 8, nv.F32, frame0=-1, clip=4), nv.E_INVALID, "clip of 4 frames")
    expect(call(2, 8, 8, nv.F32, frame0=3, clip=4), nv.E_INVALID, "clip of 4 frames")
    expect(call(2, 8, 8, nv.F32, clip=2**31), nv.E_INVALID, "clip of")
    # draws past 32-bit indexing: 22 x 4K fp32, 44 x 4K fp16, one 16K x 16K fp32 frame (even in a draw of one frame)
    expect(call(22, 2160, 3840, nv.F32, draw=22), nv.E_UNSUPPORTED, "exceeds 32-bit indexing")
    expect(call(1, 2160, 3840, nv.F32, clip=30, draw=0x7FFFFFFF), nv.E_UNSUPPORTED, "exceeds 32-bit indexing")
    expect(call(44, 2160, 3840, nv.F16, draw=44), nv.E_UNSUPPORTED, "exceeds 32-bit indexing")
    expect(call(1, 16384, 16384, nv.F32, draw=1), nv.E_UNSUPPORTED, "exceeds 32-bit indexing")
    # nothing to do is a success before any CUDA call
    assert call(0, 2160, 3840, nv.F32, clip=0, draw=22) == nv.VRGDG_OK

    inc = ctypes.c_int64(-1)
    assert lib.vrgdg_torch_randn_increment(0, ctypes.byref(inc)) == nv.VRGDG_OK and inc.value == 0
    expect(lib.vrgdg_torch_randn_increment(-1, ctypes.byref(inc)), nv.E_INVALID, "negative numel")
    expect(lib.vrgdg_torch_randn_increment(5, None), nv.E_INVALID, "null output")
    # the library-internal mode is no public seed mode
    assert lib.vrgdg_grain(src, dst, 1, 8, 8, nv.F32, ctypes.c_float(0.1), ctypes.c_float(0.5), ctypes.c_float(0.5), ctypes.c_uint64(1),
                           ctypes.c_int64(0), 4, None, None) == nv.E_INVALID


def test_noise_source_from_the_environment(pkg, monkeypatch):
    rt = pkg._runtime
    monkeypatch.delenv("VRGDG_GRAIN_NOISE", raising=False)
    assert rt.grain_noise_from_env() == "vrgdg"
    for raw, want in (("", "vrgdg"), ("vrgdg", "vrgdg"), ("torch_cuda", "torch_cuda"), (" torch_cuda ", "torch_cuda")):
        monkeypatch.setenv("VRGDG_GRAIN_NOISE", raw)
        assert rt.grain_noise_from_env() == want
    for raw in ("cpu", "TORCH", "torch"):
        monkeypatch.setenv("VRGDG_GRAIN_NOISE", raw)
        with pytest.raises(ValueError, match="vrgdg or torch_cuda"):
            rt.grain_noise_from_env()
    assert rt.NOISE_STREAMS == ("vrgdg", "torch_cuda")


def test_node_refusals_come_before_any_generator_or_device_work(pkg, monkeypatch):
    """an unknown value, and in torch_cuda mode a mini-batch draw past 32-bit indexing, raise ValueError before the CPU generator
    is drawn from and before any CUDA call or upload"""
    node = pkg.NODE_CLASS_MAPPINGS["FastFilmGrain"]()
    state = torch.get_rng_state()
    monkeypatch.setenv("VRGDG_GRAIN_NOISE", "mt19937")
    with pytest.raises(ValueError, match="VRGDG_GRAIN_NOISE=mt19937"):
        node.apply_grain(torch.zeros(1, 4, 4, 3), 0.04, 0.5, 4)
    monkeypatch.setenv("VRGDG_GRAIN_NOISE", "torch_cuda")
    clip = torch.zeros(1, 1, 1, 3).expand(30, 2160, 3840, 3)      # 30 x 4K fp32 frames without the memory
    for batch_size in (0, 22, 500):
        with pytest.raises(ValueError, match="batch_size=%d" % batch_size):
            node.apply_grain(clip, 0.04, 0.5, batch_size)
    with pytest.raises(ValueError, match="lower batch_size"):                 # 16-bit draws: 44 x 4K frames
        node.apply_grain(torch.zeros(1, 1, 1, 3, dtype=torch.float16).expand(44, 2160, 3840, 3), 0.04, 0.5, 0)
    assert torch.equal(state, torch.get_rng_state())
    types = node.INPUT_TYPES()
    assert list(types) == ["required"] and list(types["required"]) == ["images", "grain_intensity", "saturation_mix", "batch_size"]

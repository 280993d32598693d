"""Torch-stream grain (VRGDG_SEED_TORCH_PER_FRAME / _PER_CALL) without a GPU: the element -> (thread, curand4 call, float4 lane)
mapping and the Philox counter / key layout of csrc/vrgdg_math.cuh, compiled for the host (tests/hostcheck/torch_stream.cpp), against
a restatement of ATen's calc_execution_policy and distribution_elementwise_grid_stride_kernel; the C ABI's refusals, which return
before any CUDA call; and the Python argument checks."""
import ctypes
import importlib
import os
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostcheck", "torch_stream.cpp")
u32p = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")

H100_SXM_SMS, MAX_THREADS_PER_SM = 132, 2048
T_H100 = 256 * H100_SXM_SMS * (MAX_THREADS_PER_SM // 256)


@pytest.fixture(scope="module")
def ts(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("torch_stream") / "libtorch_stream.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", so], check=True)
    lib = ctypes.CDLL(so)
    lib.ts_threads.restype = ctypes.c_uint32
    lib.ts_threads.argtypes = [ctypes.c_uint64, ctypes.c_int, ctypes.c_int]
    lib.ts_sites.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, u32p, u32p, u32p]
    lib.ts_bits.argtypes = [ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, u32p]
    lib.ts_philox.argtypes = [u32p, u32p, u32p]
    lib.ts_draw_seed.restype = ctypes.c_uint64
    lib.ts_draw_seed.argtypes = [ctypes.c_uint64, ctypes.c_int64, ctypes.c_int64, ctypes.c_int]
    lib.ts_draw_base.restype = ctypes.c_uint32
    lib.ts_draw_base.argtypes = [ctypes.c_int64, ctypes.c_int64, ctypes.c_int]
    return lib


def aten_policy(numel, sms, max_threads_per_sm=MAX_THREADS_PER_SM):
    """calc_execution_policy (DistributionTemplates.h): 256-thread blocks, grid capped at SMs x (max threads per SM / 256)."""
    block = 256
    grid = min(sms * (max_threads_per_sm // block), (numel + block - 1) // block)
    return block * grid


def aten_sites(numel, T, k0, k1):
    """distribution_elementwise_grid_stride_kernel with unroll 4, iterations k0..k1-1 of every thread: thread idx starts at
    linear_index = idx and steps by 4T while linear_index < rounded_size; in iteration k its curand_normal4 lane ii writes
    li = linear_index + T*ii when li < numel.  Returns (li, k, ii, idx) of the writes, in li order."""
    rounded = ((numel - 1) // (4 * T) + 1) * 4 * T
    k = np.arange(k0, k1, dtype=np.int64)[:, None, None]
    ii = np.arange(4, dtype=np.int64)[None, :, None]
    idx = np.arange(T, dtype=np.int64)[None, None, :]
    linear_index = idx + k * 4 * T
    li = linear_index + T * ii
    ok = (linear_index < rounded) & (li < numel)
    shape = np.broadcast_shapes(k.shape, ii.shape, idx.shape)
    return tuple(np.broadcast_to(a, shape)[ok] for a in (li, k, ii, idx))


NUMELS = [1, 3, 255, 256, 257, "4T-1", "4T", "4T+1", 1920 * 1080 * 3, 3840 * 2160 * 3]


@pytest.mark.parametrize("sms", [132, 114, 1])
@pytest.mark.parametrize("numel", NUMELS, ids=str)
def test_element_mapping_is_atens_grid_stride_loop(ts, sms, numel):
    T_full = aten_policy(1 << 40, sms)
    if isinstance(numel, str):
        numel = eval(numel.replace("4T", str(4 * T_full)))
    T = aten_policy(numel, sms)
    assert ts.ts_threads(numel, sms, MAX_THREADS_PER_SM) == T
    iters = (numel - 1) // (4 * T) + 1
    step = max(1, (1 << 21) // (4 * T))                 # iterations per chunk: about 2 M elements
    seen = 0
    for k0 in range(0, iters, step):
        li, k, ii, idx = aten_sites(numel, T, k0, min(iters, k0 + step))
        n = len(li)
        assert np.array_equal(li, np.arange(seen, seen + n))    # every element is written exactly once, in li order
        gk, gii, gidx = (np.zeros(n, dtype=np.uint32) for _ in range(3))
        ts.ts_sites(seen, n, T, gk, gii, gidx)
        assert np.array_equal(gk, k) and np.array_equal(gii, ii) and np.array_equal(gidx, idx)
        seen += n
    assert seen == numel


def test_h100_thread_count(ts):
    """132 SMs x 8 blocks of 256 threads; small draws use ceil(numel / 256) blocks."""
    assert T_H100 == 270336
    assert ts.ts_threads(3840 * 2160 * 3, 132, 2048) == T_H100
    assert ts.ts_threads(17 * 23 * 3, 132, 2048) == 256 * 5
    assert ts.ts_threads(1, 132, 2048) == 256


def test_philox_known_answers(ts):
    """Random123 kat_vectors for philox4x32-10, through the in-place key schedule the torch stream uses."""
    cases = [([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
             ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
             ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0], [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1])]
    for ctr, key, want in cases:
        o = np.zeros(4, dtype=np.uint32)
        ts.ts_philox(np.array(ctr, dtype=np.uint32), np.array(key, dtype=np.uint32), o)
        assert o.tolist() == want


def test_counter_and_key_layout(ts):
    """element li reads Philox(counter {lo k, hi k, lo idx, hi idx}, key {lo seed, hi seed}) = the k-th curand4 of
    curand_init(seed, idx, 0); the four lanes of one call share the bits"""
    T = T_H100
    for seed in (0, 42, 0x7FFFFFFF, 2**64 - 1, 2**63, 0x0123456789ABCDEF):
        for li in (0, 1, T - 1, T, 3 * T + 5, 4 * T, 4 * T + 7, 9 * T + 11, 3840 * 2160 * 3 - 1):
            k, r = divmod(li, 4 * T)
            ii, idx = divmod(r, T)
            want = np.zeros(4, dtype=np.uint32)
            ts.ts_philox(np.array([k, 0, idx, 0], dtype=np.uint32), np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint32), want)
            got = np.zeros(4, dtype=np.uint32)
            ts.ts_bits(seed, li, T, got)
            assert np.array_equal(got, want), (seed, li)
            lane0 = np.zeros(4, dtype=np.uint32)
            ts.ts_bits(seed, k * 4 * T + idx, T, lane0)             # ii = 0 of the same call
            assert np.array_equal(got, lane0)


def test_draw_seeds_and_bases(ts):
    """PER_FRAME: (seed + frame0 + i) & 0x7FFFFFFF and a fresh draw per frame; PER_CALL: the seed, frames consecutive in one draw"""
    assert ts.ts_draw_seed(40, 2, 0, 2) == 42 and ts.ts_draw_seed(0x7FFFFFFF, 0, 1, 2) == 0 and ts.ts_draw_seed(5, 10**6, 3, 2) == 5 + 10**6 + 3
    assert ts.ts_draw_seed(2**64 - 1, 7, 3, 3) == 2**64 - 1
    assert ts.ts_draw_base(5, 17 * 23, 2) == 0 and ts.ts_draw_base(5, 17 * 23, 3) == 5 * 17 * 23 * 3


def _desc(nv, **kw):
    d = nv.ChainDesc()
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def test_abi_refuses_unreproducible_torch_draws_without_a_gpu(pkg):
    nv = pkg._native
    lib = nv.load_library()
    src, dst = ctypes.c_void_p(256), ctypes.c_void_p(512)          # non-null, aligned, never dereferenced
    seed, f0 = ctypes.c_uint64(42), ctypes.c_int64(0)

    def grain(B, H, W, dtype, mode):
        return lib.vrgdg_grain(src, dst, B, H, W, dtype, ctypes.c_float(0.1), ctypes.c_float(0.5), ctypes.c_float(0.5), seed, f0, mode,
                               None, None)

    def expect(rc, text):
        assert rc == nv.E_UNSUPPORTED, (rc, lib.vrgdg_last_error())
        assert text in lib.vrgdg_last_error().decode()

    # a draw whose byte extent needs 64-bit indexing: 30 x 4K x 3 fp32 elements; per frame, a 16K x 16K frame
    expect(grain(30, 2160, 3840, nv.F32, nv.SEED_TORCH_PER_CALL), "exceeds 32-bit indexing")
    expect(grain(30, 2160, 3840, nv.U8BGR, nv.SEED_TORCH_PER_CALL), "exceeds 32-bit indexing")   # bytes draw fp32 noise
    expect(grain(60, 2160, 3840, nv.F16, nv.SEED_TORCH_PER_CALL), "exceeds 32-bit indexing")
    expect(grain(1, 16384, 16384, nv.F32, nv.SEED_TORCH_PER_FRAME), "exceeds 32-bit indexing")
    out = ctypes.c_void_p(1024)
    expect(lib.vrgdg_grain_noise(out, 30, 2160, 3840, seed, f0, nv.SEED_TORCH_PER_CALL, None), "exceeds 32-bit indexing")
    expect(lib.vrgdg_grain_noise(out, 1, 16384, 16384, seed, f0, nv.SEED_TORCH_PER_FRAME, None), "exceeds 32-bit indexing")

    first = [_desc(nv, grain_enabled=1, grain_intensity=0.1, grain_sat=0.5, grain_one_minus_sat=0.5, grain_seed=1, grain_seed_mode=m,
                   stencil_op=nv.STENCIL_BOX_UNSHARP, stencil_strength=0.5) for m in (nv.SEED_TORCH_PER_FRAME, nv.SEED_TORCH_PER_CALL)]
    for d in first:
        cm = _desc(nv, **{f: getattr(d, f) for f, _ in nv.ChainDesc._fields_ if f.startswith("grain")}, colormatch_enabled=1)
        expect(lib.vrgdg_chain_apply(src, dst, 2, 64, 64, nv.F32, ctypes.byref(d), None), "first grain stage")
        expect(lib.vrgdg_chain_apply_ch(src, dst, 2, 64, 64, 3, nv.F32, ctypes.byref(d), None), "first grain stage")
        expect(lib.vrgdg_chain_apply_ext(src, dst, 2, 64, 64, nv.F32, ctypes.byref(d), None, 0, None), "first grain stage")
        scratch = ctypes.c_void_p(4096)
        expect(lib.vrgdg_chain_lab_moments(src, 2, 64, 64, nv.F32, ctypes.byref(d), ctypes.c_void_p(2048), scratch, 1 << 30, None),
               "first grain stage")
        expect(lib.vrgdg_chain_lab_moments_ext(src, 2, 64, 64, nv.F32, ctypes.byref(d), None, ctypes.c_void_p(2048), scratch, 1 << 30, None),
               "first grain stage")
        expect(lib.vrgdg_chain_cm_apply(src, dst, 2, 64, 64, nv.F32, ctypes.byref(cm), ctypes.c_void_p(2048), 1, None, 0, scratch, 1 << 30,
                                        0, None), "first grain stage")

    post = dict(stencil_op=nv.STENCIL_BOX_UNSHARP, stencil_strength=0.5, post_grain_enabled=1, post_intensity=0.1, post_sat=0.5,
                post_one_minus_sat=0.5, post_seed=7)
    expect(lib.vrgdg_chain_apply(src, dst, 2, 64, 64, nv.F32, ctypes.byref(_desc(nv, post_seed_mode=nv.SEED_TORCH_PER_CALL, **post)), None),
           "post grain takes VRGDG_SEED_TORCH_PER_FRAME")
    expect(lib.vrgdg_chain_apply(src, dst, 1, 16384, 16384, nv.F32, ctypes.byref(_desc(nv, post_seed_mode=nv.SEED_TORCH_PER_FRAME, **post)),
                                 None), "exceeds 32-bit indexing")
    # an unknown mode is still an invalid argument
    assert grain(1, 8, 8, nv.F32, 4) == nv.E_INVALID


def test_python_noise_arguments_without_a_gpu(pkg):
    vt = importlib.import_module(pkg.__name__ + ".video_tools")
    x = torch.zeros(1, 4, 4, 3)
    with pytest.raises(ValueError, match="needs a seed"):
        vt._apply_film_grain_tensor(x, 0.1, 0.5, "cuda", None, noise="torch_cuda")
    for call in (lambda: vt._apply_film_grain_tensor(x, 0.1, 0.5, "cuda", 1, noise="cpu"),
                 lambda: vt._apply_seeded_grain(x, 0.1, 0.5, 1, 0, noise="mt19937"),
                 lambda: vt._apply_effects_batch(x, {}, 0, noise="x"),
                 lambda: vt.enhance_frames([], 8, 8, {}, 0, noise="x")):
        with pytest.raises(ValueError, match="noise must be one of"):
            call()
    assert (pkg._native.SEED_TORCH_PER_FRAME, pkg._native.SEED_TORCH_PER_CALL) == (2, 3)


def test_enhance_frames_node_takes_an_optional_noise_stream(pkg):
    node = pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_EnhanceFrames"]
    types = node.INPUT_TYPES()
    assert list(types["required"]) == ["images", "sharpen_strength", "grain_intensity", "saturation_mix", "seed", "frame_start", "use_gpu"]
    choices, opts = types["optional"]["noise_stream"]
    assert choices == ["vrgdg", "torch_cuda"] and opts["default"] == "vrgdg"
    with pytest.raises(ValueError, match="noise must be one of"):
        node().enhance(torch.zeros(1, 4, 4, 3), 0.5, 0.1, 0.5, 1, 0, True, noise_stream="cpu")

"""The Video Enhance restore as one streamed, sharded kernel pass (vrgdg_restore_blend, video_enhance.restore_frames).

* k_restore against the composition it replaces: ops.resize(enhanced) -> .to(originals' dtype) -> ops.blend over the RGB of the
  originals, written into originals.clamp(0, 1) (torch.equal), and against the oracle (tests/restore_matrix.py holds the cases and
  bars; a CPU test checks that every instantiation has a case);
* the node on the reference's own outputs with small chunk caps, chunking and the placement of both batches invisible in the result;
* VRGDG_DEVICES sharding of host originals (one worker per non-empty shard, the unsharded node's tensor);
* device memory that follows the chunk, not the clip."""
import functools
import importlib
import json
import os
import threading

import pytest
import torch

import restore_matrix as rm
import video_tools_matrix as vtm
from helpers import GOLDEN, load_golden, natural_frames, t

pytestmark = pytest.mark.gpu

PKG = "comfyui-vrgamedevgirl_b200"
DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
KEY = "VRGDGVideoEnhanceRestoreOriginal"


def _ve():
    return importlib.import_module(PKG + ".video_enhance")


def _rt():
    return importlib.import_module(PKG + "._runtime")


@pytest.fixture(autouse=True)
def _env(monkeypatch):
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    monkeypatch.delenv("VRGDG_STREAM_CHUNK_BYTES", raising=False)


def _frames(B, H, W, channels, seed, dtype=torch.float32):
    """natural frames stretched past [0, 1] (the clamp is part of the result); a 4th channel of uniform values in [-0.2, 1.2)"""
    x = natural_frames(B, H, W, seed=seed) * 1.2 - 0.1
    if channels == 4:
        a = torch.rand(B, H, W, 1, generator=torch.Generator().manual_seed(seed + 1)) * 1.4 - 0.2
        x = torch.cat([x, a], dim=-1).contiguous()
    return x.to(dtype)


def _composition(ops, enh, orig, mode, roi, s, n):
    """today's restore arithmetic before the fused kernel, restated: resample, cast, blend the RGB of the first n frames, clamp"""
    H, W = int(orig.shape[1]), int(orig.shape[2])
    out = orig.clamp(0, 1)
    if n > 0:
        restored = ops.resize(enh[:n], H, W, mode, roi=roi).to(orig.dtype)
        out[:n, ..., :3] = ops.blend(orig[:n, ..., :3], restored, 1.0 - s, s)
    return out


def _diff(got, want):
    d = (got.double() - want.double()).abs()
    return "max |diff| %.3g on %d of %d elements" % (float(d.max()), int((got != want).sum()), got.numel())


@functools.lru_cache(maxsize=None)
def _case_inputs(c):
    fit, (He, We) = rm.GEOMETRIES[c.geometry]
    W = rm.WIDTHS[c.width]
    orig = _frames(rm.FRAMES, rm.HEIGHT, W, c.co, seed=W + c.co, dtype=DT[c.dtype])
    enh = _frames(rm.FRAMES, He, We, c.ce, seed=100 + He + c.ce, dtype=DT[c.dtype])
    roi = _ve()._restore_roi(We, He, W, rm.HEIGHT, fit)
    return orig, enh, roi, fit


# ---- 1. the fused kernel against the composition ------------------------------------------------------------------------------
@pytest.mark.parametrize("c", rm.CASES, ids=rm.case_id)
def test_fused_kernel_equals_the_composition(pkg, cuda_device, c):
    orig, enh, roi, _ = _case_inputs(c)
    o, e = orig.to(cuda_device), enh.to(cuda_device)
    for n in rm.N_RESTORED:
        for s in rm.STRENGTHS:
            before = pkg._native.launch_count()
            got = pkg.ops.restore_blend(e, o, c.mode, 1.0 - s, s, roi=roi, n_restored=n)
            assert pkg._native.launch_count() - before == 1
            want = _composition(pkg.ops, e, o, c.mode, roi, s, n)
            assert got.dtype == o.dtype and got.shape == o.shape and got.device == cuda_device
            assert torch.equal(got, want), (n, s, _diff(got, want))
    assert torch.equal(pkg.ops.restore_blend(e, o, c.mode, 0.5, 0.5, roi=roi), _composition(pkg.ops, e, o, c.mode, roi, 0.5, rm.FRAMES))


# ---- 2. against the oracle ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", rm.CASES, ids=rm.case_id)
def test_fused_kernel_vs_oracle(pkg, oracle, cuda_device, c):
    """oracle.restore_batch + oracle.restore_blend on the up-cast input; the restored frames are rounded to the frame dtype, as the
    reference's `restored` tensor is, and the blend once at the end"""
    orig, enh, roi, fit = _case_inputs(c)
    H, W = rm.HEIGHT, rm.WIDTHS[c.width]
    restored = oracle.restore_batch(enh.float(), W, H, fit, vtm.METHOD[c.mode]).to(orig.dtype).float()
    n, s = 2, 0.35
    want = orig.float().clamp(0, 1)
    want[:n, ..., :3] = oracle.restore_blend(orig[:n, ..., :3].float(), restored[:n], s)
    want = want.to(orig.dtype)
    got = pkg.ops.restore_blend(enh.to(cuda_device), orig.to(cuda_device), c.mode, 1.0 - s, s, roi=roi, n_restored=n).cpu()
    bar = rm.oracle_bar(c)
    if bar == 0:
        assert torch.equal(got, want), _diff(got, want)
    else:
        err = float((got.double() - want.double()).abs().max())
        assert err <= bar, (err, bar)


# ---- 3. the node on the reference's outputs, chunked ----------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [1, 2], ids=["one_frame", "two_frames"])
def test_node_on_reference_outputs_in_small_chunks(pkg, cuda_device, monkeypatch, chunk):
    g = load_golden("restore_node")
    with open(os.path.join(GOLDEN, "restore_node_cases.json")) as fh:
        cases = json.load(fh)
    node = pkg.NODE_CLASS_MAPPINGS[KEY]()
    orig, ltx = t(g["originals"]), t(g["ltx"])
    for ci, (fit, method, strength) in enumerate(cases):
        ctx = {"original_frames": orig, "source_height": 30, "source_width": 40, "frame_count": 5, "fit_mode": fit, "fps": 24.0}
        monkeypatch.delenv("VRGDG_STREAM_CHUNK_BYTES", raising=False)
        whole = node.restore(ltx, ctx, method, strength)[0]
        monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(chunk * orig[0].numel() * orig.element_size()))
        frames, n, w, h, fps = node.restore(ltx, ctx, method, strength)
        assert (n, w, h, fps) == (5, 40, 30, 24.0) and frames.device.type == "cpu" and frames.dtype == orig.dtype
        tol = 0.0 if method in ("Nearest", "Area") else 2e-6
        assert float((frames.double() - t(g["case%d" % ci]).double()).abs().max()) <= tol, (fit, method)
        assert torch.equal(frames, whole), (fit, method)


# ---- 4. chunking and placement are invisible ----------------------------------------------------------------------------------
PLACEMENTS = ["pinned", "pageable", "cuda_originals_host_enhanced", "host_originals_cuda_enhanced", "dtype_mismatch"]


@pytest.mark.parametrize("placement", PLACEMENTS)
def test_chunking_is_invisible(pkg, cuda_device, monkeypatch, placement):
    H, W = 21, 32
    fit, method, s = "Fit with letterbox (preserve all)", "Bicubic (recommended)", 0.7
    orig = _frames(7, H, W, 3, seed=5)
    enh = _frames(6, 24, 24, 3, seed=6, dtype=torch.float16 if placement == "dtype_mismatch" else torch.float32)
    if placement == "pinned":
        orig = orig.pin_memory()
    elif placement == "cuda_originals_host_enhanced":
        orig = orig.to(cuda_device)
    elif placement == "host_originals_cuda_enhanced":
        enh = enh.to(cuda_device)
    roi = _ve()._restore_roi(24, 24, W, H, fit)
    want = _composition(pkg.ops, enh.to(cuda_device), orig.to(cuda_device), "bicubic", roi, s, 6)
    results = []
    for cap in (1, 3, None):
        if cap is None:
            monkeypatch.delenv("VRGDG_STREAM_CHUNK_BYTES", raising=False)
        else:
            monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(cap * orig[0].numel() * orig.element_size()))
        got = _ve().restore_frames(orig, enh, W, H, fit, method, s)
        assert (got.device, got.dtype, got.shape) == (orig.device, orig.dtype, orig.shape)
        if orig.is_pinned():
            assert got.is_pinned()
        results.append(got)
    for got in results:
        assert torch.equal(got.to(cuda_device), want), _diff(got.to(cuda_device), want)


# ---- 5. sharding over VRGDG_DEVICES -------------------------------------------------------------------------------------------
LAYOUTS = {                                      # frames, workers on cuda:0, frames per chunk
    "uneven_small_chunks": (7, 2, 2),
    "three_workers": (7, 3, 8),
    "empty_shard": (2, 3, 8),
}
SH, SW = 21, 32


def _cards():
    return [torch.device("cuda", i) for i in range(torch.cuda.device_count()) if tuple(torch.cuda.get_device_capability(i)) == (9, 0)]


def _node(pkg, orig, enh):
    ctx = {"original_frames": orig, "source_height": SH, "source_width": SW, "frame_count": int(orig.shape[0]),
           "fit_mode": "Fit with letterbox (preserve all)", "fps": 24.0}
    return pkg.NODE_CLASS_MAPPINGS[KEY]().restore(enh, ctx, "Bicubic (recommended)", 0.7)[0]


def _trace(monkeypatch):
    rt = _rt()
    log = {"sharded": [], "streams": []}
    sharded, stream = rt.stream_frames_sharded, rt.stream_frames

    def traced_sharded(src, make_fn, chunk, out_device, devices, out=None):
        log["sharded"].append([torch.device(d) for d in devices])
        return sharded(src, make_fn, chunk, out_device, devices, out=out)

    def traced_stream(src, fn, chunk, out_device, device=None, **kw):
        log["streams"].append((threading.current_thread().name, device, int(src.shape[0])))
        return stream(src, fn, chunk, out_device, device, **kw)
    monkeypatch.setattr(rt, "stream_frames_sharded", traced_sharded)
    monkeypatch.setattr(rt, "stream_frames", traced_stream)
    return log


def _compare_sharded(pkg, monkeypatch, orig, enh, devices):
    """the node unsharded (one stream_frames call in this thread), then over `devices` (a list patched in as devices_from_env, or a
    VRGDG_DEVICES string): one worker per non-empty shard, no thread left behind, the same tensor with the same placement"""
    main = threading.current_thread().name
    log = _trace(monkeypatch)
    one = _node(pkg, orig, enh)
    assert not log["sharded"] and [name for name, _, _ in log["streams"]] == [main]
    if isinstance(devices, str):
        monkeypatch.setenv("VRGDG_DEVICES", devices)
        cards = _rt().devices_from_env()
    else:
        monkeypatch.setattr(_ve(), "devices_from_env", lambda: list(devices))
        cards = list(devices)
    log["sharded"].clear()
    log["streams"].clear()
    threads = threading.active_count()
    got = _node(pkg, orig, enh)
    assert threading.active_count() == threads, "a worker thread outlived the call"
    assert log["sharded"] == [cards]
    n = int(orig.shape[0])
    if len(cards) == 1:
        assert log["streams"] == [(main, cards[0], n)]
    else:
        calls = sorted((int(name.rsplit("-", 1)[1]), dev, k) for name, dev, k in log["streams"] if name.startswith("vrgdg-shard-"))
        want = [(d, b - a) for d, (a, b) in zip(cards, _rt().shard_plan(n, len(cards))) if b > a]
        assert [(dev, k) for _, dev, k in calls] == want
        assert all(name != main for name, _, _ in log["streams"])
    assert (got.device, got.dtype, got.shape, got.is_pinned()) == (one.device, one.dtype, one.shape, one.is_pinned())
    assert not torch.equal(one, orig.clamp(0, 1)), "the node left the frames unrestored"
    assert torch.equal(got, one)


def _shard_inputs(monkeypatch, n, chunk, dtype, pinned):
    orig = _frames(n, SH, SW, 3, seed=11, dtype=dtype)
    orig = orig.pin_memory() if pinned else orig
    enh = _frames(max(1, n - 1), 24, 24, 3, seed=12, dtype=dtype)     # one frame short: the last original is only clamped
    monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(chunk * orig[0].numel() * orig.element_size()))
    return orig, enh


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_workers_on_one_card_match_the_unsharded_node(pkg, cuda_device, monkeypatch, layout, pinned, dtype):
    n, workers, chunk = LAYOUTS[layout]
    orig, enh = _shard_inputs(monkeypatch, n, chunk, DT[dtype], pinned)
    _compare_sharded(pkg, monkeypatch, orig, enh, [cuda_device] * workers)


@pytest.mark.parametrize("layout", ["uneven_small_chunks", "empty_shard"])
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_every_card_matches_the_unsharded_node(pkg, cuda_device, monkeypatch, layout, pinned):
    cards = _cards()
    if len(cards) < 2:
        pytest.skip("one compute-capability-9.0 device visible; the one-card tests cover the sharded path")
    n, chunk = (2 * len(cards) + 1, 2) if layout == "uneven_small_chunks" else (len(cards) - 1, 8)
    orig, enh = _shard_inputs(monkeypatch, n, chunk, torch.float32, pinned)
    _compare_sharded(pkg, monkeypatch, orig, enh, cards)


@pytest.mark.parametrize("value", ["0", "all"])
def test_real_vrgdg_devices_values(pkg, cuda_device, monkeypatch, value):
    orig, enh = _shard_inputs(monkeypatch, 7, 2, torch.float32, False)
    _compare_sharded(pkg, monkeypatch, orig, enh, value)


def test_cuda_originals_are_one_call_on_their_device(pkg, cuda_device, monkeypatch):
    orig, enh = _shard_inputs(monkeypatch, 7, 2, torch.float32, False)
    log = _trace(monkeypatch)
    monkeypatch.setattr(_ve(), "devices_from_env", lambda: [cuda_device] * 2)
    before = pkg._native.launch_count()
    got = _node(pkg, orig.to(cuda_device), enh)
    assert pkg._native.launch_count() - before == 1 and not log["sharded"]
    assert got.device == cuda_device and torch.equal(got.cpu(), _node(pkg, orig, enh))


# ---- 6. device memory follows the chunk -----------------------------------------------------------------------------------------
def test_device_memory_is_bounded_by_the_chunk_not_the_clip(pkg, cuda_device, monkeypatch):
    """48 x 540p fp32 host originals (~300 MB) restored in two-frame chunks.  Allocated device memory at any time: the three
    pipeline slots of stream_frames (depth 2 + 1), the chunk's output and its enhanced slice.  Resampling the whole clip at once and
    blending into a clamped copy took about four times the clip."""
    B, H, W, He, We = 48, 540, 960, 288, 512
    g = torch.Generator().manual_seed(3)
    orig = torch.rand(B, H, W, 3, generator=g) * 1.2 - 0.1
    enh = torch.rand(B, He, We, 3, generator=g)
    frame, enh_frame = H * W * 3 * 4, He * We * 3 * 4
    monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(2 * frame))
    torch.cuda.synchronize(cuda_device)
    torch.cuda.reset_peak_memory_stats(cuda_device)
    base = torch.cuda.memory_allocated(cuda_device)
    out = _ve().restore_frames(orig, enh, W, H, "Stretch to dimensions", "Bicubic (recommended)", 0.7)
    torch.cuda.synchronize(cuda_device)
    grew = torch.cuda.max_memory_allocated(cuda_device) - base
    chunk = 2 * frame
    bound = 3 * chunk + chunk + 2 * enh_frame + (4 << 20)   # slots, output, enhanced slice, allocator rounding
    clip = B * frame
    assert grew <= bound and grew < clip // 4, "device memory grew by %.1f MB (bound %.1f MB, clip %.1f MB)" % (grew / 1e6, bound / 1e6, clip / 1e6)
    for k in (0, 23, 47):                          # spot frames against the one-launch result on the device
        want = pkg.ops.restore_blend(enh[k:k + 1].to(cuda_device), orig[k:k + 1].to(cuda_device), "bicubic", 1.0 - 0.7, 0.7)
        assert torch.equal(out[k:k + 1], want.cpu())

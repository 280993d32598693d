"""The Video Enhance resample helpers streamed and sharded (video_enhance._resize_batch / _restore_batch on run_frames).

* every mode x fit x dtype x channel count x ROI, upscaled and downscaled, from pageable host, pinned host and CUDA batches, in
  one-frame and uneven chunks: torch.equal to one whole-batch ops.resize launch on the device with the same plan;
* stream_frames / stream_frames_sharded with out_frame_shape directly: two workers on one card, every visible card, the chunked
  CUDA-source branch and the `out=` check;
* VRGDG_DEVICES sharding of host batches (one worker per non-empty shard, on its device; none for a CUDA batch);
* device memory that follows the chunk, not the clip."""
import importlib
import itertools
import threading

import pytest
import torch

import video_tools_matrix as vtm
from helpers import natural_frames

pytestmark = pytest.mark.gpu

PKG = "comfyui-vrgamedevgirl_b200"
DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
FITS = {"stretch": "Stretch to dimensions", "crop": "Crop to fill", "letterbox": "Fit with letterbox (preserve all)"}
SRC_H, SRC_W, FRAMES = 37, 53, 5
TARGETS = {"up": (90, 64), "down": (29, 23)}                          # (target width, target height) from 53 x 37 frames
SOURCES = ("pageable", "pinned", "cuda")


def _ve():
    return importlib.import_module(PKG + ".video_enhance")


def _rt():
    return importlib.import_module(PKG + "._runtime")


@pytest.fixture(autouse=True)
def _env(monkeypatch):
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    monkeypatch.delenv("VRGDG_STREAM_CHUNK_BYTES", raising=False)


def _frames(B, H, W, channels, seed, dtype):
    """natural frames stretched past [0, 1] (the clamp is part of the result); a 4th channel that the resample drops"""
    x = natural_frames(B, H, W, seed=seed) * 1.2 - 0.1
    if channels == 4:
        x = torch.cat([x, torch.rand(B, H, W, 1, generator=torch.Generator().manual_seed(seed + 1))], dim=-1).contiguous()
    return x.to(dtype)


def _place(x, source, dev):
    return x.pin_memory() if source == "pinned" else x.to(dev) if source == "cuda" else x


def _one_launch(pkg, x, dev, tw, th, fit, mode, roi=None):
    """today's arithmetic: the whole batch on the device, one ops.resize launch with _resize_batch's plan"""
    ve = _ve()
    x0, y0, sw, sh = roi if roi is not None else (0, 0, int(x.shape[2]), int(x.shape[1]))
    res, off = ve._resize_plan(sw, sh, tw, th, fit)
    ow, oh = ve._output_size(res, off, tw, th, fit)
    return pkg.ops.resize(x.to(dev), oh, ow, mode, roi=(x0, y0, sw, sh), resampled=res, offset=off)


def _diff(got, want):
    d = (got.double() - want.double()).abs()
    return "max |diff| %.3g on %d of %d elements" % (float(d.max()), int((got != want).sum()), got.numel())


def _check_streamed(pkg, monkeypatch, x, dev, want, call):
    """call() on every source placement and chunking; each result torch.equal to `want` with the source's device and dtype"""
    frame = max(x[0].numel(), want[0].numel()) * x.element_size()
    for source, cap in itertools.product(SOURCES, (1, 2, None)):       # one-frame chunks, 2 + 2 + 1, the default (one chunk)
        if cap is None:
            monkeypatch.delenv("VRGDG_STREAM_CHUNK_BYTES", raising=False)
        else:
            monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(cap * frame))
        src = _place(x, source, dev)
        before = pkg._native.launch_count()
        got = call(src)
        launches = pkg._native.launch_count() - before
        assert (got.device, got.dtype, got.shape) == (src.device, src.dtype, want.shape), (source, cap)
        if source == "cuda":
            assert launches == 1, "a CUDA batch is one launch whatever the chunk cap"
        else:
            assert launches == (-(-FRAMES // cap) if cap else 1), (source, cap, launches)
        if source == "pinned":
            assert got.is_pinned()
        assert torch.equal(got.to(dev), want), (source, cap, _diff(got.to(dev), want))


@pytest.mark.parametrize("dtype", list(DT))
@pytest.mark.parametrize("fit", list(FITS))
@pytest.mark.parametrize("mode", vtm.RESIZE_MODES)
def test_resize_batch_streamed_equals_one_launch(pkg, cuda_device, monkeypatch, mode, fit, dtype):
    ve = _ve()
    for ch, (geo, (tw, th)) in itertools.product((3, 4), TARGETS.items()):
        x = _frames(FRAMES, SRC_H, SRC_W, ch, seed=tw + ch, dtype=DT[dtype])
        want = _one_launch(pkg, x, cuda_device, tw, th, FITS[fit], mode)
        _check_streamed(pkg, monkeypatch, x, cuda_device, want,
                        lambda src: ve._resize_batch(src, tw, th, FITS[fit], vtm.METHOD[mode]))


@pytest.mark.parametrize("dtype", list(DT))
@pytest.mark.parametrize("mode", vtm.RESIZE_MODES)
def test_restore_batch_roi_streamed_equals_one_launch(pkg, cuda_device, monkeypatch, mode, dtype):
    """_restore_batch of letterboxed working frames: the content rectangle is the ROI of every chunk, upscaled and downscaled back"""
    ve = _ve()
    for ch, (sw, sh) in itertools.product((3, 4), ((53, 37), (160, 120))):
        x = _frames(FRAMES, 80, 80, ch, seed=sw + ch, dtype=DT[dtype])
        roi = ve._restore_roi(80, 80, sw, sh, FITS["letterbox"])
        assert roi[1] > 0 and roi[3] < 80
        want = _one_launch(pkg, x, cuda_device, sw, sh, FITS["stretch"], mode, roi=roi)
        _check_streamed(pkg, monkeypatch, x, cuda_device, want,
                        lambda src: ve._restore_batch(src, sw, sh, FITS["letterbox"], vtm.METHOD[mode]))


# ---- the runtime directly -------------------------------------------------------------------------------------------------------
def _cards():
    return [torch.device("cuda", i) for i in range(torch.cuda.device_count()) if tuple(torch.cuda.get_device_capability(i)) == (9, 0)]


def _resize_fn(oh, ow):
    """make_fn for stream_frames_sharded: a bicubic resample of each chunk to oh x ow"""
    ops = importlib.import_module(PKG + ".ops")
    return lambda dev: (lambda f, first: ops.resize(f, oh, ow, "bicubic"))


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("layout", [(7, 2, 2), (7, 3, 8), (2, 3, 8)], ids=["uneven_small_chunks", "three_workers", "empty_shard"])
def test_workers_on_one_card_through_stream_frames_sharded(pkg, cuda_device, monkeypatch, layout, pinned):
    n, workers, chunk = layout
    x = _frames(n, 27, 48, 3, seed=n + workers, dtype=torch.float32)
    x = x.pin_memory() if pinned else x
    oh, ow = 54, 96
    monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(chunk * oh * ow * 3 * 4))
    want = pkg.ops.resize(x.to(cuda_device), oh, ow, "bicubic")
    threads = threading.active_count()
    got = _rt().stream_frames_sharded(x, _resize_fn(oh, ow), 0, "cpu", [cuda_device] * workers, out_frame_shape=(oh, ow, 3))
    assert threading.active_count() == threads
    assert got.shape == (n, oh, ow, 3) and got.device.type == "cpu" and got.is_pinned()
    assert torch.equal(got.to(cuda_device), want)
    out = torch.empty(n, oh, ow, 3)
    assert _rt().stream_frames_sharded(x, _resize_fn(oh, ow), 0, "cpu", [cuda_device] * workers, out=out, out_frame_shape=(oh, ow, 3)) is out
    assert torch.equal(out.to(cuda_device), want)
    with pytest.raises(ValueError, match="result's shape"):
        _rt().stream_frames_sharded(x, _resize_fn(oh, ow), 0, "cpu", [cuda_device] * workers, out=x.clone(), out_frame_shape=(oh, ow, 3))


def test_every_card_through_stream_frames_sharded(pkg, cuda_device, monkeypatch):
    cards = _cards()
    if len(cards) < 2:
        pytest.skip("one compute-capability-9.0 device visible; the one-card tests cover the sharded path")
    n, oh, ow = 2 * len(cards) + 1, 54, 96
    x = _frames(n, 27, 48, 4, seed=3, dtype=torch.float32)
    monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(2 * oh * ow * 3 * 4))
    got = _rt().stream_frames_sharded(x, _resize_fn(oh, ow), 0, "cpu", cards, out_frame_shape=(oh, ow, 3))
    assert torch.equal(got.to(cuda_device), pkg.ops.resize(x.to(cuda_device), oh, ow, "bicubic"))


@pytest.mark.parametrize("out_device", ["cpu", "cuda"])
def test_chunked_cuda_source_with_another_frame_shape(pkg, cuda_device, out_device):
    x = _frames(7, 27, 48, 3, seed=4, dtype=torch.bfloat16).to(cuda_device)
    want = pkg.ops.resize(x, 20, 30, "area")
    dev = cuda_device if out_device == "cuda" else torch.device("cpu")
    got = _rt().stream_frames(x, lambda f, i: pkg.ops.resize(f, 20, 30, "area"), 3, dev, out_frame_shape=(20, 30, 3))
    assert got.shape == (7, 20, 30, 3) and got.dtype == x.dtype and got.device == dev
    assert torch.equal(got.to(cuda_device), want)


def test_out_of_the_wrong_shape_is_refused(pkg, cuda_device):
    x = _frames(3, 27, 48, 3, seed=5, dtype=torch.float32)
    fn = lambda f, i: pkg.ops.resize(f, 20, 30, "nearest")             # noqa: E731
    with pytest.raises(ValueError, match="result's shape"):
        _rt().stream_frames(x, fn, 0, "cpu", cuda_device, out=torch.empty_like(x), out_frame_shape=(20, 30, 3))
    out = torch.empty(3, 20, 30, 3)
    assert _rt().stream_frames(x, fn, 0, "cpu", cuda_device, out=out, out_frame_shape=(20, 30, 3)) is out
    assert torch.equal(out, pkg.ops.resize(x.to(cuda_device), 20, 30, "nearest").cpu())


# ---- VRGDG_DEVICES ----------------------------------------------------------------------------------------------------------------
def _trace(monkeypatch):
    rt = _rt()
    log = {"sharded": [], "streams": []}
    sharded, stream = rt.stream_frames_sharded, rt.stream_frames

    def traced_sharded(src, make_fn, chunk, out_device, devices, out=None, **kw):
        log["sharded"].append([torch.device(d) for d in devices])
        return sharded(src, make_fn, chunk, out_device, devices, out=out, **kw)

    def traced_stream(src, fn, chunk, out_device, device=None, **kw):
        log["streams"].append((threading.current_thread().name, device, int(src.shape[0])))
        return stream(src, fn, chunk, out_device, device, **kw)
    monkeypatch.setattr(rt, "stream_frames_sharded", traced_sharded)
    monkeypatch.setattr(rt, "stream_frames", traced_stream)
    return log


def _call(x):
    return _ve()._resize_batch(x, 96, 54, FITS["crop"], "Bicubic (recommended)")


def _compare_sharded(monkeypatch, x, devices):
    """_resize_batch unsharded (one stream_frames call in this thread), then over `devices` (a list patched in as devices_from_env,
    or a VRGDG_DEVICES string): one worker per non-empty shard on that shard's device, no thread left behind, the same tensor"""
    main = threading.current_thread().name
    log = _trace(monkeypatch)
    one = _call(x)
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
    got = _call(x)
    assert threading.active_count() == threads, "a worker thread outlived the call"
    assert log["sharded"] == [cards]
    n = int(x.shape[0])
    if len(cards) == 1:
        assert log["streams"] == [(main, cards[0], n)]
    else:
        calls = sorted((int(name.rsplit("-", 1)[1]), dev, k) for name, dev, k in log["streams"] if name.startswith("vrgdg-shard-"))
        want = [(d, b - a) for d, (a, b) in zip(cards, _rt().shard_plan(n, len(cards))) if b > a]
        assert [(dev, k) for _, dev, k in calls] == want
        assert all(name != main for name, _, _ in log["streams"])
    assert (got.device, got.dtype, got.shape, got.is_pinned()) == (one.device, one.dtype, one.shape, one.is_pinned())
    assert torch.equal(got, one)


def _shard_input(monkeypatch, n, chunk, pinned, dtype=torch.float32):
    x = _frames(n, 27, 48, 3, seed=11, dtype=dtype)
    monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(chunk * 54 * 96 * 3 * x.element_size()))
    return x.pin_memory() if pinned else x


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("layout", [(7, 2, 2), (7, 3, 8), (2, 3, 8)], ids=["uneven_small_chunks", "three_workers", "empty_shard"])
def test_resize_batch_workers_on_one_card(pkg, cuda_device, monkeypatch, layout, pinned):
    n, workers, chunk = layout
    _compare_sharded(monkeypatch, _shard_input(monkeypatch, n, chunk, pinned, torch.bfloat16), [cuda_device] * workers)


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_resize_batch_every_card(pkg, cuda_device, monkeypatch, pinned):
    cards = _cards()
    if len(cards) < 2:
        pytest.skip("one compute-capability-9.0 device visible; the one-card tests cover the sharded path")
    _compare_sharded(monkeypatch, _shard_input(monkeypatch, 2 * len(cards) + 1, 2, pinned), cards)


@pytest.mark.parametrize("value", ["0", "all"])
def test_real_vrgdg_devices_values(pkg, cuda_device, monkeypatch, value):
    _compare_sharded(monkeypatch, _shard_input(monkeypatch, 7, 2, False), value)


def test_cuda_batches_are_one_launch_and_never_shard(pkg, cuda_device, monkeypatch):
    x = _shard_input(monkeypatch, 7, 2, False)
    log = _trace(monkeypatch)
    monkeypatch.setattr(_ve(), "devices_from_env", lambda: [cuda_device] * 2)
    before = pkg._native.launch_count()
    got = _call(x.to(cuda_device))
    assert pkg._native.launch_count() - before == 1 and not log["sharded"]
    assert log["streams"] == [(threading.current_thread().name, cuda_device, 7)]
    assert got.device == cuda_device and torch.equal(got.cpu(), _call(x))
    monkeypatch.undo()
    monkeypatch.setenv("VRGDG_DEVICES", "not-a-card")                  # a CUDA batch does not read the variable
    assert torch.equal(_call(x.to(cuda_device)), got)
    with pytest.raises(ValueError, match="VRGDG_DEVICES=not-a-card"):
        _call(x)


# ---- device memory follows the chunk --------------------------------------------------------------------------------------------
def test_device_memory_is_bounded_by_the_chunk_not_the_clip(pkg, cuda_device, monkeypatch):
    """48 x 540p -> 1080p fp32 host frames (~300 MB in, ~1.2 GB out) in two-frame chunks.  Allocated device memory at any time: the
    three pipeline slots of input frames and at most three chunks of results waiting for their download.  Before, the whole clip
    and its whole result were on the card."""
    B, H, W, Ho, Wo = 48, 540, 960, 1080, 1920
    x = torch.rand(B, H, W, 3, generator=torch.Generator().manual_seed(3)) * 1.2 - 0.1
    frame, out_frame = H * W * 3 * 4, Ho * Wo * 3 * 4
    monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(2 * out_frame))
    torch.cuda.synchronize(cuda_device)
    torch.cuda.reset_peak_memory_stats(cuda_device)
    base = torch.cuda.memory_allocated(cuda_device)
    out = _ve()._resize_batch(x, Wo, Ho, FITS["stretch"], "Bicubic (recommended)")
    torch.cuda.synchronize(cuda_device)
    grew = torch.cuda.max_memory_allocated(cuda_device) - base
    bound = 4 * 2 * (frame + out_frame)                              # four chunks of input + output
    clip = B * out_frame
    assert grew < bound and grew < clip // 4, "device memory grew by %.1f MB (bound %.1f MB, output clip %.1f MB)" % (
        grew / 1e6, bound / 1e6, clip / 1e6)
    assert out.shape == (B, Ho, Wo, 3) and out.device.type == "cpu"
    for k in (0, 23, 47):                                            # spot frames against the one-launch result on the device
        want = pkg.ops.resize(x[k:k + 1].to(cuda_device), Ho, Wo, "bicubic")
        assert torch.equal(out[k:k + 1], want.cpu())

"""The streamed Video Enhance resample helpers without a GPU: what video_enhance._resize_batch / _restore_batch hand to run_frames
(the planned output frame shape and the one resample plan of every chunk), how stream_frames sizes its pipeline chunks when the
result frames have another shape, that out_frame_shape=None reaches exactly the calls it reached before the option existed, and
that the helpers' errors and VRGDG_DEVICES refusals come where they did."""
import importlib

import pytest
import torch

import video_tools_matrix as vtm

PKG = "comfyui-vrgamedevgirl_b200"
FITS = ("Stretch to dimensions", "Crop to fill", "Fit with letterbox (preserve all)")
CUDA0 = torch.device("cuda", 0)


def _ve():
    return importlib.import_module(PKG + ".video_enhance")


def _rt():
    return importlib.import_module(PKG + "._runtime")


class Stop(Exception):
    """raised by a stand-in to end a call before it would need a device"""


@pytest.fixture(autouse=True)
def _env(monkeypatch):
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    monkeypatch.delenv("VRGDG_STREAM_CHUNK_BYTES", raising=False)


def _capture(monkeypatch):
    """run_frames of video_enhance replaced by a recorder; the compute device is cuda:0 without asking CUDA"""
    ve, calls = _ve(), []

    def run_frames(images, make_fn, chunk, out_device, device, devices, **kw):
        calls.append(dict(images=images, make_fn=make_fn, chunk=chunk, out_device=torch.device(out_device), device=device,
                          devices=devices, **kw))
        return "result"
    monkeypatch.setattr(ve, "run_frames", run_frames)
    monkeypatch.setattr(ve, "compute_device", lambda images=None: CUDA0)
    return calls


def _resize_args(pkg, monkeypatch, make_fn, frames):
    """the arguments fn(frames, first) hands to ops.resize"""
    seen = []

    def resize(images, out_h, out_w, mode, roi=None, resampled=None, offset=(0, 0)):
        seen.append((images, out_h, out_w, mode, roi, resampled, offset))
        return torch.zeros(int(images.shape[0]), out_h, out_w, 3, dtype=images.dtype)
    monkeypatch.setattr(pkg.ops, "resize", resize)
    out = make_fn(CUDA0)(frames, 3)
    assert len(seen) == 1 and seen[0][0] is frames
    return out, seen[0][1:]


@pytest.mark.parametrize("fit", FITS)
def test_resize_batch_hands_run_frames_the_planned_output_shape(pkg, oracle, monkeypatch, fit):
    """for each fit mode and some sizes: the out_frame_shape is the shape the reference produces (oracle, nearest), and every chunk
    is one ops.resize call with the unchanged plan"""
    ve = _ve()
    calls = _capture(monkeypatch)
    for (sw, sh), (tw, th) in [((53, 37), (90, 29)), ((53, 37), (64, 64)), ((53, 37), (80, 80)), ((40, 30), (17, 33)), ((9, 31), (31, 9))]:
        for ch in (3, 4):
            x = torch.rand(2, sh, sw, ch)
            assert ve._resize_batch(x, tw, th, fit, "Nearest") == "result"
            c = calls.pop()
            want = oracle.resize_batch(x[..., :3], tw, th, fit, "Nearest")
            assert c["out_frame_shape"] == tuple(want.shape[1:]), (sw, sh, tw, th, fit)
            assert c["images"] is x and c["chunk"] == 0 and c["out_device"] == x.device and c["device"] == CUDA0 and c["devices"] is None
            res, off = ve._resize_plan(sw, sh, tw, th, fit)
            out, args = _resize_args(pkg, monkeypatch, c["make_fn"], x[:1])
            assert args == (want.shape[1], want.shape[2], "nearest", (0, 0, sw, sh), res, off)
            assert tuple(out.shape[1:]) == c["out_frame_shape"]


@pytest.mark.parametrize("method", list(vtm.METHOD.values()))
def test_restore_batch_hands_over_the_letterbox_roi(pkg, monkeypatch, method):
    """_restore_batch streams the same way: the source size as the output frame, the letterbox content (or the whole working frame
    for the other fit modes) as the ROI of every chunk's resample"""
    ve = _ve()
    calls = _capture(monkeypatch)
    mode = {v: k for k, v in vtm.METHOD.items()}[method]
    x = torch.rand(2, 80, 80, 3)                                       # an 80 x 80 working frame
    for fit in FITS:
        ve._restore_batch(x, 53, 37, fit, method)
        c = calls.pop()
        assert c["out_frame_shape"] == (37, 53, 3) and c["images"] is x and c["devices"] is None
        roi = (0, 12, 80, 56) if fit == FITS[2] else (0, 0, 80, 80)    # the letterbox content is rows 12 .. 67
        assert ve._restore_roi(80, 80, 53, 37, fit) == roi
        _, args = _resize_args(pkg, monkeypatch, c["make_fn"], x)
        assert args == (37, 53, mode, roi, (53, 37), (0, 0))


def test_errors_come_before_any_device_work(pkg, monkeypatch):
    ve = _ve()

    def fail(*a, **k):
        raise AssertionError("device work before the argument check")
    for name in ("compute_device", "devices_from_env", "run_frames", "upload"):
        monkeypatch.setattr(ve, name, fail)
    monkeypatch.setenv("VRGDG_DEVICES", "not-a-card")
    x = torch.rand(3, 6, 8, 3)
    for bad in (x[:0], x[0], x[None]):
        with pytest.raises(ValueError, match="non-empty IMAGE batch"):
            ve._resize_batch(bad, 8, 8, "Stretch to dimensions", "Nearest")
        for fit in FITS:
            with pytest.raises(ValueError, match="non-empty IMAGE batch"):
                ve._restore_batch(bad, 8, 8, fit, "Nearest")


def test_malformed_vrgdg_devices_raises_only_when_a_host_batch_streams(pkg, monkeypatch):
    ve = _ve()
    calls = _capture(monkeypatch)
    x = torch.rand(2, 6, 8, 3)
    monkeypatch.setenv("VRGDG_DEVICES", "not-a-card")
    with pytest.raises(ValueError, match="VRGDG_DEVICES=not-a-card"):
        ve._resize_batch(x, 16, 12, "Crop to fill", "Bilinear")
    with pytest.raises(ValueError, match="VRGDG_DEVICES=not-a-card"):
        ve._restore_batch(x, 16, 12, "Fit with letterbox (preserve all)", "Bilinear")
    assert calls == []
    # a batch that does not live on the host never reads the variable (a meta tensor stands in for a CUDA one here)
    m = torch.empty(2, 6, 8, 3, device="meta")
    ve._resize_batch(m, 16, 12, "Crop to fill", "Bilinear")
    assert calls.pop()["devices"] is None
    monkeypatch.setenv("VRGDG_DEVICES", "")
    ve._resize_batch(x, 16, 12, "Crop to fill", "Bilinear")
    assert calls.pop()["devices"] is None


def test_resize_batch_shards_host_batches_over_vrgdg_devices(pkg, monkeypatch):
    ve = _ve()
    calls = _capture(monkeypatch)
    monkeypatch.setattr(ve, "devices_from_env", lambda: [CUDA0, CUDA0])
    x = torch.rand(5, 6, 8, 4)
    ve._resize_batch(x, 16, 12, "Stretch to dimensions", "Area")
    c = calls.pop()
    assert c["devices"] == [CUDA0, CUDA0] and c["out_frame_shape"] == (12, 16, 3)


def _stream_until_chunking(monkeypatch, src, **kw):
    """stream_frames on a host source up to its pipeline_chunk call: (frames asked for, frame bytes it was sized on)"""
    rt, seen = _rt(), []

    def pipeline_chunk(chunk, frame_bytes, cap=None):
        seen.append((chunk, frame_bytes))
        raise Stop
    monkeypatch.setattr(rt, "pipeline_chunk", pipeline_chunk)
    with pytest.raises(Stop):
        rt.stream_frames(src, lambda f, i: f, 0, "cpu", CUDA0, **kw)
    return seen.pop()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_chunks_are_sized_on_the_larger_frame(monkeypatch, dtype):
    es = torch.empty((), dtype=dtype).element_size()
    pipeline_chunk = _rt().pipeline_chunk
    up = torch.empty(6, 540, 960, 3, dtype=dtype)                     # 540p -> 1080p: the result frame is 4 x the source frame
    assert _stream_until_chunking(monkeypatch, up, out_frame_shape=(1080, 1920, 3)) == (6, 1080 * 1920 * 3 * es)
    down = torch.empty(6, 1080, 1920, 4, dtype=dtype)                 # RGBA 1080p -> RGB 720p: the source frame is the larger
    assert _stream_until_chunking(monkeypatch, down, out_frame_shape=(720, 1280, 3)) == (6, 1080 * 1920 * 4 * es)
    assert _stream_until_chunking(monkeypatch, up) == (6, 540 * 960 * 3 * es)
    cap = 2 * 1080 * 1920 * 3 * es                                    # two result frames: two frames per chunk, not eight
    assert pipeline_chunk(48, 1080 * 1920 * 3 * es, cap) == 2 and pipeline_chunk(48, 540 * 960 * 3 * es, cap) == 8


def test_empty_host_batches_take_the_result_shape(monkeypatch):
    rt = _rt()
    x = torch.zeros(0, 6, 8, 4, dtype=torch.bfloat16)
    never = lambda f, i: pytest.fail("fn called on an empty batch")   # noqa: E731
    same = rt.stream_frames(x, never, 0, "cpu", CUDA0)
    assert same.shape == x.shape and same.dtype == x.dtype
    other = rt.stream_frames(x, never, 0, "cpu", CUDA0, out_frame_shape=(12, 16, 3))
    assert other.shape == (0, 12, 16, 3) and other.dtype == x.dtype and other.device.type == "cpu"


def _record(monkeypatch, name):
    rt, seen = _rt(), []

    def rec(*args, **kw):
        seen.append((args, kw))
        return "result"
    monkeypatch.setattr(rt, name, rec)
    return seen


def test_none_reaches_the_calls_of_before(monkeypatch):
    """run_frames and stream_frames_sharded without out_frame_shape pass exactly the arguments they passed before it existed;
    with it, they pass it on and nothing else changes"""
    rt = _rt()
    real_sharded = rt.stream_frames_sharded
    streams, sharded = _record(monkeypatch, "stream_frames"), _record(monkeypatch, "stream_frames_sharded")
    x = torch.zeros(4, 6, 8, 3)
    fn = lambda f, i: f                                                # noqa: E731
    made = []

    def make_fn(dev):
        made.append(dev)
        return fn
    assert rt.run_frames(x, make_fn, 3, "cpu", CUDA0, None) == "result"
    assert streams.pop() == ((x, fn, 3, "cpu", CUDA0), {}) and made.pop() == CUDA0
    assert rt.run_frames(x, make_fn, 3, "cpu", CUDA0, [CUDA0, CUDA0]) == "result"
    assert sharded.pop() == ((x, make_fn, 3, "cpu", [CUDA0, CUDA0]), {})
    assert rt.run_frames(x, make_fn, 3, "cpu", CUDA0, None, out_frame_shape=(2, 2, 3)) == "result"
    assert streams.pop() == ((x, fn, 3, "cpu", CUDA0), {"out_frame_shape": (2, 2, 3)})
    assert rt.run_frames(x, make_fn, 3, "cpu", CUDA0, [CUDA0], out_frame_shape=(2, 2, 3)) == "result"
    assert sharded.pop() == ((x, make_fn, 3, "cpu", [CUDA0]), {"out_frame_shape": (2, 2, 3)})
    assert rt.run_frames(x, make_fn, 3, CUDA0, CUDA0, [CUDA0, CUDA0]) == "result"          # a CUDA result never shards
    assert streams.pop() == ((x, fn, 3, CUDA0, CUDA0), {}) and not sharded
    # stream_frames_sharded's one-device call
    assert real_sharded(x, make_fn, 3, "cpu", ["cuda:0"]) == "result"
    assert streams.pop() == ((x, fn, 3, torch.device("cpu"), CUDA0), {"out": None})
    assert real_sharded(x, make_fn, 3, "cpu", ["cuda:0"], out_frame_shape=(2, 2, 3)) == "result"
    assert streams.pop() == ((x, fn, 3, torch.device("cpu"), CUDA0), {"out": None, "out_frame_shape": (2, 2, 3)})

"""VRGDG_DEVICES on every frame node: a host IMAGE batch sharded over several workers gives what the node gives with it unset.

Every node here works per frame or keys its work by the absolute frame index, and the split adds no arithmetic, so each sharded
result must be torch.equal to the unsharded one.  Two or three workers on one card come from patching the node modules'
devices_from_env (the parser rejects a repeated index); the cases over every visible card skip when only one is visible.  The CPU
test at the end keeps every IMAGE node of NODE_CLASS_MAPPINGS either in NODES or on the explicit EXEMPT list."""
import importlib
import os
import shutil
import threading

import pytest
import torch

from helpers import LUTS, natural_frames

H, W = 48, 96                                   # wide enough for the TMA tile path
LUT = "B200 Vintage 33.cube"
MODULES = ("filter_nodes", "lut_nodes", "chain_nodes")
DTYPES = {"f32": torch.float32, "f16": torch.float16}
# frames, workers on cuda:0, frames per chunk
LAYOUTS = {
    "uneven_small_chunks": (7, 2, 2),           # shards of 4 and 3 frames in chunks of 2
    "three_workers": (7, 3, 8),                 # shards of 3, 2 and 2 frames
    "empty_shard": (2, 3, 8),                   # fewer frames than workers
}

# the sharded nodes: key -> run(node, frames, reference, chunk) -> IMAGE.  `chunk` goes to the batch_size widget where there is one;
# VRGDG_STREAM_CHUNK_BYTES cuts the other nodes' batches the same way.
NODES = {
    "FastFilmGrain": lambda n, x, ref, chunk: n.apply_grain(x, 0.05, 0.4, chunk)[0],
    "ColorMatchToReference": lambda n, x, ref, chunk: n.match_color(x, ref, 0.8, chunk)[0],
    "FastUnsharpSharpen": lambda n, x, ref, chunk: n.apply_unsharp(x, 0.5, False)[0],
    "FastLaplacianSharpen": lambda n, x, ref, chunk: n.apply_laplacian(x, 0.5, True)[0],
    "FastSobelSharpen": lambda n, x, ref, chunk: n.apply_sobel(x, 0.5, False)[0],
    "VRGDG_LUTS": lambda n, x, ref, chunk: n.apply_lut(x, LUT, "auto", 7.5)[0],
    "VRGDG_MakeLUT": lambda n, x, ref, chunk: n.create_and_apply(x, "#0b1d51, #1f6aa5, #f3d27a", "shard", 17, "auto", 10.0)[0],
    "VRGDG_B200_HistogramColorMatch": lambda n, x, ref, chunk: n.match_histogram(x, ref, 0.8, chunk)[0],
    "VRGDG_B200_TemporalSharpen": lambda n, x, ref, chunk: n.sharpen(x, 0.7, chunk)[0],
    "VRGDG_B200_PostChain": lambda n, x, ref, chunk: n.apply_chain(x, 0.04, 0.5, 0.8, LUT, 10.0, "unsharp", 0.5, False, chunk,
                                                                   reference_image=ref)[0],
    "VRGDG_B200_EnhanceFrames": lambda n, x, ref, chunk: n.enhance(x, 0.5, 0.05, 0.3, 42, 3, True)[0],
}
# Nodes that do not shard.  VRGDGVideoEnhanceRestoreOriginal takes two batches of different sizes and does not stream them.
# VRGDGStandaloneVideoEnhancer has no IMAGE input (the guard below never selects it); it is listed so that the list names every
# graph node the feature leaves out, not because an IMAGE path of it opts out.
EXEMPT = {"VRGDGVideoEnhanceRestoreOriginal", "VRGDGStandaloneVideoEnhancer"}


@pytest.fixture(autouse=True)
def luts_dir(pkg, monkeypatch, tmp_path):
    """The LUT nodes read and write LUTS_DIR: here a copy of the shipped table in tmp_path, so VRGDG_MakeLUT writes nothing into the
    package.  VRGDG_DEVICES and the chunk cap start unset."""
    shutil.copy(os.path.join(LUTS, LUT), tmp_path / LUT)
    monkeypatch.setattr(importlib.import_module(pkg.__name__ + ".lut_nodes"), "LUTS_DIR", str(tmp_path))
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    monkeypatch.delenv("VRGDG_STREAM_CHUNK_BYTES", raising=False)
    return tmp_path


def _cards():
    return [torch.device("cuda", i) for i in range(torch.cuda.device_count()) if tuple(torch.cuda.get_device_capability(i)) == (9, 0)]


def _frames(dtype, n, seed=11, pinned=False):
    x = natural_frames(n, H, W, seed=seed).to(dtype)
    return x.pin_memory() if pinned else x


def _chunked(monkeypatch, x, chunk):
    monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(chunk * x[0].numel() * x.element_size()))


def _shard(pkg, monkeypatch, devices):
    """A string goes through the real parser as VRGDG_DEVICES; a list is handed to every node module as its devices_from_env()."""
    if isinstance(devices, str):
        monkeypatch.setenv("VRGDG_DEVICES", devices)
        return
    for m in MODULES:
        monkeypatch.setattr(importlib.import_module(pkg.__name__ + "." + m), "devices_from_env", lambda: list(devices))


def _run(pkg, key, x, ref, chunk):
    torch.manual_seed(1234)                     # FastFilmGrain and the PostChain node draw their grain seed from torch's generator
    return NODES[key](pkg.NODE_CLASS_MAPPINGS[key](), x, ref, chunk)


def _trace(pkg, monkeypatch):
    """Record every stream_frames_sharded call (its device list) and every stream_frames call (thread name, device, frames).
    run_frames and the shard workers look both names up in _runtime at call time, so the wrappers see what the nodes really run."""
    rt = importlib.import_module(pkg.__name__ + "._runtime")
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


def _workers(log):
    """(device, frames) of every shard worker's stream_frames call, in shard order."""
    calls = [(int(name.rsplit("-", 1)[1]), dev, n) for name, dev, n in log["streams"] if name.startswith("vrgdg-shard-")]
    return [(dev, n) for _, dev, n in sorted(calls, key=lambda c: c[0])]


def _compare(pkg, monkeypatch, key, x, ref, chunk, devices):
    """The node with VRGDG_DEVICES unset (the single-device stream_frames call, no shard), then sharded over `devices`: one worker per
    non-empty shard on the shard's device for a host batch with a host result, none otherwise; same tensor, same placement, no thread
    left behind."""
    rt = importlib.import_module(pkg.__name__ + "._runtime")
    main = threading.current_thread().name
    log = _trace(pkg, monkeypatch)
    one = _run(pkg, key, x, ref, chunk)
    assert not log["sharded"] and all(name == main for name, _, _ in log["streams"])
    if x.device.type == "cpu":
        assert len(log["streams"]) == 1, "the unsharded node did not stream its host batch once"
    _shard(pkg, monkeypatch, devices)
    cards = rt.devices_from_env() if isinstance(devices, str) else [torch.device(d) for d in devices]
    log["sharded"].clear()
    log["streams"].clear()
    threads = threading.active_count()
    got = _run(pkg, key, x, ref, chunk)
    assert threading.active_count() == threads, "a worker thread outlived the call"
    if x.device.type == "cpu" and got.device.type == "cpu":
        assert log["sharded"] == [cards], "%s did not hand its host batch to stream_frames_sharded" % key
        n = int(x.shape[0])
        if len(cards) == 1:                     # one device: stream_frames_sharded's single-device call, in this thread
            assert log["streams"] == [(main, cards[0], n)]
        else:
            want = [(d, b - a) for d, (a, b) in zip(cards, rt.shard_plan(n, len(cards))) if b > a]
            assert _workers(log) == want, "%s: shard workers %s, expected %s" % (key, _workers(log), want)
            assert all(name != main for name, _, _ in log["streams"])
    else:
        assert not log["sharded"] and not _workers(log), "%s sharded a CUDA batch or a CUDA result" % key
    assert (got.device, got.dtype, got.shape, got.is_pinned()) == (one.device, one.dtype, one.shape, one.is_pinned())
    if x.shape[0] > 1 or key != "VRGDG_B200_TemporalSharpen":    # a one-frame clip is its own neighbour: the temporal unsharp keeps it
        assert not torch.equal(one, x), "%s left the frames unchanged" % key
    assert torch.equal(got, one), key
    return got, one


@pytest.mark.gpu
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("key", list(NODES))
def test_workers_on_one_card_match_the_unsharded_node(pkg, cuda_device, monkeypatch, key, dtype, pinned, layout):
    n, workers, chunk = LAYOUTS[layout]
    x = _frames(DTYPES[dtype], n, pinned=pinned)
    _chunked(monkeypatch, x, chunk)
    _compare(pkg, monkeypatch, key, x, _frames(DTYPES[dtype], 1, seed=99), chunk, [cuda_device] * workers)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["uneven_small_chunks", "empty_shard"])
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("key", list(NODES))
def test_every_card_matches_the_unsharded_node(pkg, cuda_device, monkeypatch, key, dtype, pinned, layout):
    cards = _cards()
    if len(cards) < 2:
        pytest.skip("one compute-capability-9.0 device visible; the one-card tests cover the sharded path")
    n, chunk = (2 * len(cards) + 1, 2) if layout == "uneven_small_chunks" else (len(cards) - 1, 8)
    x = _frames(DTYPES[dtype], n, pinned=pinned)
    _chunked(monkeypatch, x, chunk)
    _compare(pkg, monkeypatch, key, x, _frames(DTYPES[dtype], 1, seed=99), chunk, cards)


@pytest.mark.gpu
@pytest.mark.parametrize("value", ["0", "all"])
@pytest.mark.parametrize("key", list(NODES))
def test_real_vrgdg_devices_values(pkg, cuda_device, monkeypatch, key, value):
    x = _frames(torch.float32, 7)
    _chunked(monkeypatch, x, 2)
    _compare(pkg, monkeypatch, key, x, _frames(torch.float32, 1, seed=99), 2, value)


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(NODES))
def test_cuda_batches_keep_the_single_device_call(pkg, cuda_device, monkeypatch, key):
    x = _frames(torch.float32, 7).to(cuda_device)
    got, _ = _compare(pkg, monkeypatch, key, x, _frames(torch.float32, 1, seed=99).to(cuda_device), 2, [cuda_device] * 2)
    assert got.device == cuda_device


@pytest.mark.gpu
def test_sharded_grain_advances_the_generator_as_one_call(pkg, cuda_device, monkeypatch):
    x = _frames(torch.float32, 7)
    node = pkg.FastFilmGrain()
    torch.manual_seed(77)
    one = node.apply_grain(x, 0.05, 0.4, 2)[0]
    state = torch.get_rng_state()
    _shard(pkg, monkeypatch, [cuda_device] * 3)
    log = _trace(pkg, monkeypatch)
    torch.manual_seed(77)
    got = node.apply_grain(x, 0.05, 0.4, 2)[0]
    assert _workers(log) == [(cuda_device, 3), (cuda_device, 2), (cuda_device, 2)]
    assert torch.equal(torch.get_rng_state(), state)
    assert torch.equal(got, one)


@pytest.mark.gpu
@pytest.mark.parametrize("key", list(NODES))
def test_malformed_vrgdg_devices_is_an_error_for_host_batches(pkg, cuda_device, monkeypatch, key):
    monkeypatch.setenv("VRGDG_DEVICES", "0,x")
    with pytest.raises(ValueError, match="'x' is not a device index"):
        _run(pkg, key, _frames(torch.float32, 3), _frames(torch.float32, 1, seed=99), 2)


@pytest.mark.gpu
@pytest.mark.parametrize("n_ref, workers, chunk", [(7, 2, 2), (7, 3, 1), (1, 2, 1)],
                         ids=["ref_per_frame_2_workers", "ref_per_frame_3_workers", "batch_size_1_2_workers"])
def test_color_match_reference_per_frame_and_scratch_per_worker(pkg, cuda_device, monkeypatch, n_ref, workers, chunk):
    # n_ref == B: each worker slices the reference sums by absolute frame index, across shard boundaries inside the batch.
    # batch_size 1, two workers on one card: a scratch shared by the workers would be handed back and forth between them.
    x = _frames(torch.float32, 7)
    _compare(pkg, monkeypatch, "ColorMatchToReference", x, _frames(torch.float32, n_ref, seed=99), chunk, [cuda_device] * workers)


@pytest.mark.gpu
def test_temporal_sharpen_sees_its_neighbours_across_shard_edges(pkg, cuda_device, monkeypatch):
    x = _frames(torch.float32, 9)               # shards [0,3) [3,6) [6,9) in chunks of 2: each edge falls between two chunks
    got, one = _compare(pkg, monkeypatch, "VRGDG_B200_TemporalSharpen", x, None, 2, [cuda_device] * 3)
    for edge in (3, 6):
        assert torch.equal(got[edge - 1:edge + 1], one[edge - 1:edge + 1])
    node = pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_TemporalSharpen"]()
    assert not torch.equal(node.sharpen(x[3:6], 0.7, 2)[0][0], one[3]), "frame 3 does not depend on frame 2: the edge test is void"


@pytest.mark.gpu
@pytest.mark.parametrize("workers", [2, 3])
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
def test_lut_node_shards_rgba_frames(pkg, cuda_device, monkeypatch, pinned, workers):
    rgb = natural_frames(7, H, W, seed=11)
    x = torch.cat([rgb, torch.linspace(0, 1, 7).view(7, 1, 1, 1).expand(7, H, W, 1)], dim=-1).contiguous()
    x = x.pin_memory() if pinned else x
    _chunked(monkeypatch, x, 2)
    _compare(pkg, monkeypatch, "VRGDG_LUTS", x, None, 2, [cuda_device] * workers)


@pytest.mark.gpu
def test_make_lut_shards_and_writes_only_to_its_luts_dir(pkg, cuda_device, monkeypatch, luts_dir):
    shipped = sorted(os.listdir(LUTS))
    x = _frames(torch.float32, 7)
    _chunked(monkeypatch, x, 2)
    _compare(pkg, monkeypatch, "VRGDG_MakeLUT", x, None, 2, [cuda_device] * 2)
    made = pkg.VRGDG_MakeLUT().create_and_apply(x, "teal, orange", "shard", 17, "auto", 10.0)
    assert os.path.dirname(made[2]) == str(luts_dir) and os.path.isfile(made[2])
    assert sorted(os.listdir(LUTS)) == shipped


def test_every_image_node_shards_or_is_exempt(pkg):
    def takes_image(cls):
        return any(isinstance(spec, tuple) and spec and spec[0] == "IMAGE"
                   for group in cls.INPUT_TYPES().values() for spec in group.values())
    keys = set(pkg.NODE_CLASS_MAPPINGS)
    assert set(NODES) <= keys and EXEMPT <= keys and not set(NODES) & EXEMPT
    missing = {k for k in keys if takes_image(pkg.NODE_CLASS_MAPPINGS[k])} - set(NODES) - EXEMPT
    assert not missing, "IMAGE nodes that neither shard host batches over VRGDG_DEVICES nor are exempt: %s" % sorted(missing)

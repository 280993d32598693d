"""Histogram colour match against a reference clip on the GPU.  vrgdg_histmatch_apply_refs is torch.equal to the three calls it
replaces (counts of the frames and of the reference frames, tables with n_ref = B, the apply pass) on every dtype, reference size and
strength, and to the specification oracle; VRGDG_B200_HistogramColorMatch with n_ref == B equals the single-reference node run frame
by frame, whatever the chunks, workers and devices; and the reference clip no longer has to fit on the card."""
import importlib
import threading

import pytest
import torch

from helpers import natural_frames

pytestmark = pytest.mark.gpu

DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
STRENGTHS = (1.0, 0.35)
KEY = "VRGDG_B200_HistogramColorMatch"


def _clip(B, H, W, seed):
    """B reference frames that differ from each other (gain and offset per frame), so a pairing mistake changes the result"""
    x = natural_frames(B, H, W, seed=seed)
    gain = torch.linspace(0.45, 0.9, B).view(B, 1, 1, 1)
    return (x * gain + (1.0 - gain) * 0.5 * torch.tensor([0.9, 0.5, 0.2])).clamp(0, 1)


def _three_calls(ops, x, refs, t):
    return ops.histmatch_apply(x, ops.histmatch_tables(ops.hist_counts(x), ops.hist_counts(refs)), t, 1.0 - t)


# ---- library ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", list(DT))
def test_entry_equals_counts_tables_apply(pkg, cuda_device, dtype):
    """B = 5 frames of 72 x 93; reference frames smaller, equal and larger, odd sizes included; strengths 1 and 0.35"""
    ops = pkg.ops
    x = natural_frames(5, 72, 93, seed=1).to(cuda_device, DT[dtype])
    x[0, :2, :5] = torch.tensor([0.0, 1.0, 0.5], device=cuda_device, dtype=DT[dtype])      # exact bin edges / extremes
    scratch = None
    for size in ((33, 47), (72, 93), (131, 257), (1, 1)):
        refs = _clip(5, *size, seed=2).to(cuda_device, DT[dtype])
        for t in STRENGTHS:
            got, scratch = ops.histmatch_apply_refs(x, refs, t, 1.0 - t, scratch=scratch)
            assert torch.equal(got, _three_calls(ops, x, refs, t)), (size, t)
    # the scratch was reused: it was large enough after the first call
    assert scratch.numel() >= int(pkg._native.load_library().vrgdg_histmatch_refs_scratch_bytes(5))


def test_entry_on_one_frame_empty_batches_and_in_place(pkg, cuda_device):
    ops = pkg.ops
    x = natural_frames(3, 40, 56, seed=3).to(cuda_device)
    refs = _clip(3, 24, 30, seed=4).to(cuda_device)
    one, _ = ops.histmatch_apply_refs(x[1:2], refs[1:2], 0.8, 0.2)
    assert torch.equal(one, _three_calls(ops, x[1:2], refs[1:2], 0.8))
    empty, _ = ops.histmatch_apply_refs(x[:0], refs[:0], 0.8, 0.2)
    assert empty.shape == (0, 40, 56, 3)
    # the call is stream ordered (counts before the apply pass), so the C entry point may write over its input
    want = _three_calls(ops, x, refs, 0.8)
    y = x.clone()
    lib = pkg._native.load_library()
    nv = pkg._native
    scratch = torch.empty(int(lib.vrgdg_histmatch_refs_scratch_bytes(3)), dtype=torch.uint8, device=cuda_device)
    with torch.cuda.device(cuda_device):
        nv.check(lib.vrgdg_histmatch_apply_refs(nv.ptr(y), nv.ptr(y), 3, 40, 56, nv.F32, nv.ptr(refs), 24, 30, pkg.ops._f32(0.8),
                                                pkg.ops._f32(0.2), nv.ptr(scratch), scratch.numel(), nv.stream_ptr(cuda_device)))
    assert torch.equal(y, want)


def test_entry_counts_more_frames_than_one_launch_holds(pkg, cuda_device):
    """the counts kernel takes one frame per grid row (at most 65535): a larger batch is counted in slices, and gives what two calls
    over the two halves give"""
    B = 65535 + 7
    g = torch.Generator(device=cuda_device).manual_seed(20)
    x = torch.rand(B, 2, 3, 3, device=cuda_device, generator=g)
    refs = torch.rand(B, 3, 2, 3, device=cuda_device, generator=g) * 0.5 + 0.25
    got, _ = pkg.ops.histmatch_apply_refs(x, refs, 1.0, 0.0)
    for a, b in ((0, 65535), (65535, B)):
        part, _ = pkg.ops.histmatch_apply_refs(x[a:b], refs[a:b], 1.0, 0.0)
        assert torch.equal(got[a:b], part), (a, b)
    assert not torch.equal(got, x)


def test_entry_fp32_equals_the_specification_oracle(pkg, cuda_device, oracle):
    x = natural_frames(4, 48, 61, seed=5)
    refs = _clip(4, 37, 29, seed=6)
    for t in STRENGTHS:
        got, _ = pkg.ops.histmatch_apply_refs(x.to(cuda_device), refs.to(cuda_device), t, 1.0 - t)
        assert torch.equal(got.cpu(), oracle.hist_match(x, refs, t)), t


def test_entry_matching_a_clip_to_itself_is_the_identity(pkg, cuda_device):
    x = natural_frames(3, 270, 480, seed=7).to(cuda_device)
    same, _ = pkg.ops.histmatch_apply_refs(x, x, 1.0, 0.0)
    assert float((same - x).abs().max()) <= 1e-6                 # the plateau rule of the inverse CDF, up to hist_map's rounding


def test_entry_on_4k_frames_with_1080p_references(pkg, cuda_device):
    x = natural_frames(2, 2160, 3840, seed=8, device=cuda_device)
    refs = _clip(2, 1080, 1920, seed=9).to(cuda_device)
    got, _ = pkg.ops.histmatch_apply_refs(x, refs, 0.35, 0.65)
    assert torch.equal(got, _three_calls(pkg.ops, x, refs, 0.35))


def test_ops_refuses_a_reference_clip_that_does_not_match(pkg, cuda_device):
    x = natural_frames(3, 16, 16, seed=10).to(cuda_device)
    for bad in (x[:2], x.half(), x.cpu()):
        with pytest.raises((ValueError, RuntimeError), match="ref_frames"):
            pkg.ops.histmatch_apply_refs(x, bad, 1.0, 0.0)


# ---- the node -------------------------------------------------------------------------------------------------------------------
def _per_frame(pkg, x, refs, t):
    """what a user runs today: one single-reference node call per frame"""
    node = pkg.NODE_CLASS_MAPPINGS[KEY]()
    return torch.cat([node.match_histogram(x[i:i + 1], refs[i:i + 1], t, 1)[0].to(x.device) for i in range(x.shape[0])])


@pytest.mark.parametrize("dtype", ["f32", "f16"])
def test_node_with_a_reference_clip_equals_the_single_reference_node_per_frame(pkg, oracle, monkeypatch, cuda_device, dtype):
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    monkeypatch.delenv("VRGDG_STREAM_CHUNK_BYTES", raising=False)
    x = natural_frames(7, 40, 56, seed=11).to(DT[dtype])
    refs = _clip(7, 30, 44, seed=12)                                   # fp32 references: converted to the frames' dtype per chunk
    t = 0.8
    want = _per_frame(pkg, x, refs, t)
    if dtype == "f32":
        assert torch.equal(want, oracle.hist_match(x, refs, t))
    node = pkg.NODE_CLASS_MAPPINGS[KEY]()
    for batch_size in (1, 3, 0):
        for frames_dev in ("cpu", "cuda"):
            for refs_dev in ("cpu", "cuda"):
                got = node.match_histogram(x.to(frames_dev), refs.to(refs_dev), t, batch_size)[0]
                assert got.device.type == frames_dev and torch.equal(got.cpu(), want), (batch_size, frames_dev, refs_dev)
    # pipeline chunks smaller than batch_size cut a host batch further; the pairing holds there too
    monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(2 * x[0].numel() * x.element_size()))
    assert torch.equal(node.match_histogram(x, refs, t, 0)[0], want)


def test_node_with_a_clip_of_one_repeated_frame_equals_the_single_reference_node(pkg, monkeypatch, cuda_device):
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    node = pkg.NODE_CLASS_MAPPINGS[KEY]()
    for dt in (torch.float32, torch.bfloat16):
        x = natural_frames(6, 36, 50, seed=13).to(dt)
        one = _clip(1, 28, 34, seed=14)                                 # fp32: the node converts it to the frames' dtype
        want = node.match_histogram(x, one, 0.35, 4)[0]
        assert torch.equal(node.match_histogram(x, one.expand(6, -1, -1, -1).contiguous(), 0.35, 4)[0], want)
        assert torch.equal(node.match_histogram(x.to(cuda_device), one.repeat(6, 1, 1, 1).to(cuda_device), 0.35, 4)[0].cpu(), want)


def _shard(pkg, monkeypatch, devices):
    monkeypatch.setattr(importlib.import_module(pkg.__name__ + ".chain_nodes"), "devices_from_env", lambda: list(devices))


@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("workers, batch_size", [(2, 2), (3, 1), (3, 8)])
def test_workers_on_one_card_match_the_unsharded_node(pkg, monkeypatch, cuda_device, workers, batch_size, pinned):
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    x = natural_frames(7, 48, 96, seed=15)
    refs = _clip(7, 40, 64, seed=16)
    x, refs = (x.pin_memory(), refs.pin_memory()) if pinned else (x, refs)
    node = pkg.NODE_CLASS_MAPPINGS[KEY]()
    one = node.match_histogram(x, refs, 0.8, batch_size)[0]
    _shard(pkg, monkeypatch, [cuda_device] * workers)
    threads = threading.active_count()
    got = node.match_histogram(x, refs, 0.8, batch_size)[0]
    assert threading.active_count() == threads, "a worker thread outlived the call"
    assert got.device.type == "cpu" and torch.equal(got, one)
    assert torch.equal(one, _per_frame(pkg, x, refs, 0.8))


def test_every_card_matches_the_unsharded_node(pkg, monkeypatch, cuda_device):
    cards = [torch.device("cuda", i) for i in range(torch.cuda.device_count()) if tuple(torch.cuda.get_device_capability(i)) == (9, 0)]
    if len(cards) < 2:
        pytest.skip("one compute-capability-9.0 device visible; the one-card tests cover the sharded path")
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    n = 2 * len(cards) + 1
    x = natural_frames(n, 48, 96, seed=17)
    refs = _clip(n, 40, 64, seed=18)
    node = pkg.NODE_CLASS_MAPPINGS[KEY]()
    one = node.match_histogram(x, refs, 0.8, 2)[0]
    monkeypatch.setenv("VRGDG_DEVICES", "all")
    assert torch.equal(node.match_histogram(x, refs, 0.8, 2)[0], one)
    refs_far = refs.to(cards[-1])                                       # a reference clip on another card than the frames' chunks
    assert torch.equal(node.match_histogram(x, refs_far, 0.8, 2)[0], one)


def test_node_device_memory_follows_the_chunk_not_the_reference_clip(pkg, monkeypatch, cuda_device):
    """96 host 540p fp32 frames in two-frame chunks against 96 host 1080p fp32 reference frames (2.4 GB): the device peak stays
    below four chunks of frames, reference frames and results"""
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    monkeypatch.delenv("VRGDG_STREAM_CHUNK_BYTES", raising=False)
    g = torch.Generator().manual_seed(19)
    x = torch.rand(96, 540, 960, 3, generator=g)
    refs = torch.rand(96, 1080, 1920, 3, generator=g) * 0.8
    clip_bytes = refs.numel() * refs.element_size()
    chunk_bytes = 2 * (2 * x[0].numel() + refs[0].numel()) * 4          # frames, results and reference frames of one chunk
    node = pkg.NODE_CLASS_MAPPINGS[KEY]()
    node.match_histogram(x[:6], refs[:6], 0.8, 2)                       # warm-up: kernels loaded, pinned staging buffers cached
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    got = node.match_histogram(x, refs, 0.8, 2)[0]
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print("device peak %.1f MB, four chunks %.1f MB, reference clip %.1f MB" % (peak / 1e6, 4 * chunk_bytes / 1e6, clip_bytes / 1e6))
    assert peak < 4 * chunk_bytes < clip_bytes / 4
    assert torch.equal(got[-3:], _per_frame(pkg, x[-3:], refs[-3:], 0.8))

"""In-process sharding of host frames (stream_frames_sharded, PostChain(devices=...), VRGDG_DEVICES on the chain nodes).

The split adds no arithmetic (grain is keyed by the absolute frame index, colour-match statistics are per frame, the reference
statistics are copied), so every sharded result must be torch.equal to one device's.  On one GPU the workers share cuda:0, each
with its own upload / download streams and colour-match scratch; the multi-device cases run when more than one device of compute
capability 9.0 is visible and skip otherwise."""
import importlib
import os
import threading

import pytest
import torch

from helpers import LUTS, natural_frames

pytestmark = pytest.mark.gpu

H, W = 48, 96                                   # wide enough for the TMA tile path
LUT = "B200 Vintage 33.cube"
GRAIN = dict(intensity=0.04, saturation_mix=0.5, seed=42)
CHAINS = ("grain", "grain_cm_lut_unsharp", "unsharp_post_grain")
DTYPES = {"f32": torch.float32, "f16": torch.float16, "u8": torch.uint8}
# frames, workers on cuda:0, chunk_frames, first_frame
ONE_CARD = {
    "uneven_small_chunks": (7, 2, 2, 5),        # shards of 4 and 3 frames in chunks of 2, a clip that does not start at frame 0
    "three_workers": (7, 3, 8, 0),              # shards of 3, 2 and 2 frames
    "empty_shard": (1, 2, 8, 3),                # fewer frames than workers
}


def _cards():
    return [torch.device("cuda", i) for i in range(torch.cuda.device_count()) if tuple(torch.cuda.get_device_capability(i)) == (9, 0)]


def _frames(dtype, n, seed=11):
    x = natural_frames(n, H, W, seed=seed)
    return (x * 255).round().to(torch.uint8) if dtype == torch.uint8 else x.to(dtype)


def _chain(pkg, kind, dtype, **where):
    nv = pkg._native
    if kind == "grain":
        return pkg.chain.PostChain(grain=GRAIN, **where)
    if kind == "unsharp_post_grain":            # the standalone enhancer's effect chain
        return pkg.chain.PostChain(stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5, border=nv.BORDER_ZERO),
                                   post_grain=dict(intensity=0.05, saturation_mix=0.3, seed=7, seed_mode=nv.SEED_PER_FRAME), **where)
    lut = pkg.VRGDG_LUTS._parse_cube_file(os.path.join(LUTS, LUT))
    return pkg.chain.PostChain(grain=GRAIN, colormatch=dict(reference_image=_frames(dtype, 1, seed=99), strength=0.8),
                               lut=dict(lut_data=lut, strength=10.0), stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), **where)


def _check(pkg, kind, dtype, pinned, n, devices, chunk, first):
    x = _frames(DTYPES[dtype], n)
    if pinned:
        x = x.pin_memory()
    one = _chain(pkg, kind, DTYPES[dtype], device=devices[0]).run_host(x, chunk_frames=chunk, first_frame=first)
    threads = threading.active_count()
    sharded = _chain(pkg, kind, DTYPES[dtype], devices=devices).run_host(x, chunk_frames=chunk, first_frame=first)
    assert threading.active_count() == threads
    assert sharded.device.type == "cpu" and sharded.dtype == x.dtype and sharded.shape == x.shape
    assert sharded.is_pinned() == one.is_pinned()
    assert not torch.equal(one, x), "the chain left the frames unchanged"
    assert torch.equal(sharded, one)


@pytest.mark.parametrize("layout", list(ONE_CARD))
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("kind", CHAINS)
def test_workers_on_one_card_match_one_device(pkg, cuda_device, kind, dtype, pinned, layout):
    n, workers, chunk, first = ONE_CARD[layout]
    _check(pkg, kind, dtype, pinned, n, [cuda_device] * workers, chunk, first)


@pytest.mark.parametrize("layout", ["uneven_small_chunks", "empty_shard"])
@pytest.mark.parametrize("pinned", [True, False], ids=["pinned", "pageable"])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("kind", CHAINS)
def test_every_card_matches_one_device(pkg, cuda_device, kind, dtype, pinned, layout):
    cards = _cards()
    if len(cards) < 2:
        pytest.skip("one compute-capability-9.0 device visible; the one-card tests cover the sharded path")
    n, chunk, first = (2 * len(cards) + 1, 2, 5) if layout == "uneven_small_chunks" else (len(cards) - 1, 8, 3)
    _check(pkg, kind, dtype, pinned, n, cards, chunk, first)


def test_shards_see_absolute_frame_indices_in_their_own_threads(pkg, cuda_device):
    rt = importlib.import_module(pkg.__name__ + "._runtime")
    x = natural_frames(7, 8, 16, seed=4)
    made, calls, lock = [], [], threading.Lock()

    def make_fn(dev):
        made.append(dev)

        def fn(frames, first):
            with lock:
                calls.append((threading.get_ident(), int(first), int(frames.shape[0]), torch.cuda.current_device()))
            idx = torch.arange(first, first + frames.shape[0], device=frames.device, dtype=frames.dtype)
            return frames + idx.view(-1, 1, 1, 1)                           # frame j comes back as x[j] + j
        return fn
    threads = threading.active_count()
    out = rt.stream_frames_sharded(x, make_fn, 2, torch.device("cpu"), [cuda_device] * 3)
    assert threading.active_count() == threads
    assert made == [cuda_device] * 3
    assert torch.equal(out, x + torch.arange(7, dtype=x.dtype).view(-1, 1, 1, 1))
    assert all(c[3] == cuda_device.index for c in calls)
    by_thread = {}
    for ident, first, n, _ in calls:
        by_thread.setdefault(ident, []).append((first, n))
    assert threading.get_ident() not in by_thread
    # shards [0,3), [3,5), [5,7) in chunks of at most 2 frames, one worker thread each
    assert sorted(sorted(v) for v in by_thread.values()) == [[(0, 2), (2, 1)], [(3, 2)], [(5, 2)]]


def test_a_failing_shard_is_raised_after_every_worker_finished(pkg, cuda_device):
    rt = importlib.import_module(pkg.__name__ + "._runtime")

    class ShardFailure(RuntimeError):
        pass
    x = natural_frames(7, 8, 16, seed=5).pin_memory()
    out = torch.zeros_like(x).pin_memory()
    made = []

    def make_fn(dev):
        made.append(dev)
        if len(made) == 2:
            def boom(frames, first):
                raise ShardFailure("shard 1 fails at frame %d" % first)
            return boom
        return lambda frames, first: frames * 2
    threads = threading.active_count()
    with pytest.raises(ShardFailure, match="frame 3"):
        rt.stream_frames_sharded(x, make_fn, 2, torch.device("cpu"), [cuda_device] * 3, out=out)
    assert threading.active_count() == threads
    assert torch.equal(out[:3], x[:3] * 2) and torch.equal(out[5:], x[5:] * 2)    # the other shards ran to the end before the raise


def test_sharded_run_host_fills_a_given_result(pkg, cuda_device):
    x = _frames(torch.float32, 5).pin_memory()
    chain = _chain(pkg, "grain_cm_lut_unsharp", torch.float32, devices=[cuda_device, cuda_device])
    out = torch.empty_like(x).pin_memory()
    assert chain.run_host(x, chunk_frames=2, out=out) is out
    assert torch.equal(out, _chain(pkg, "grain_cm_lut_unsharp", torch.float32, device=cuda_device).run_host(x, chunk_frames=2))
    with pytest.raises(ValueError):
        chain.run_host(x, out=torch.empty((4,) + tuple(x.shape[1:])))


def test_cuda_frames_keep_the_single_device_call(pkg, cuda_device):
    x = _frames(torch.float32, 3)
    chain = _chain(pkg, "grain_cm_lut_unsharp", torch.float32, devices=[cuda_device, cuda_device])
    single = _chain(pkg, "grain_cm_lut_unsharp", torch.float32, device=cuda_device)
    assert torch.equal(chain(x.to(cuda_device)), single(x.to(cuda_device)))
    assert torch.equal(chain.run_host(x.to(cuda_device)).cpu(), single(x.to(cuda_device)).cpu())


# ---- the nodes: VRGDG_DEVICES ------------------------------------------------------------------------------------------------
def _node_outputs(pkg, x, ref):
    torch.manual_seed(1234)                     # the PostChain node draws its grain seed from torch's generator
    chain = pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_PostChain"]().apply_chain(x, 0.04, 0.5, 0.8, LUT, 10.0, "unsharp", 0.5, False, 2,
                                                                           reference_image=ref)[0]
    enhancer = pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_EnhanceFrames"]()
    return chain, enhancer.enhance(x, 0.5, 0.05, 0.3, 42, 3, True)[0], enhancer.enhance(x, 0.0, 0.05, 0.3, 42, 3, True)[0]


@pytest.mark.parametrize("mode", ["two_workers_on_0", "0", "all"])
def test_nodes_shard_host_batches_bit_identically(pkg, cuda_device, monkeypatch, mode):
    nodes = importlib.import_module(pkg.__name__ + ".chain_nodes")
    x, ref = _frames(torch.float32, 7), _frames(torch.float32, 1, seed=99)
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    want = _node_outputs(pkg, x, ref)
    if mode == "two_workers_on_0":
        # VRGDG_DEVICES rejects a repeated index, so the two workers on the one card are handed to the nodes past the parser
        monkeypatch.setattr(nodes, "devices_from_env", lambda: [cuda_device, cuda_device])
    else:
        monkeypatch.setenv("VRGDG_DEVICES", mode)
    got = _node_outputs(pkg, x, ref)
    for g, w in zip(got, want):
        assert g.device.type == "cpu" and torch.equal(g, w)
    assert not torch.equal(got[0], x) and not torch.equal(got[1], x) and not torch.equal(got[2], x)

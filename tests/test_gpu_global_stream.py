"""FastFilmGrain with VRGDG_GRAIN_NOISE=torch_cuda on the GPU: the node equals the reference's loop run on CUDA frames
(oracle.film_grain, whose torch.randn_like draws from the device's global generator) and leaves that generator's offset where the
reference leaves it; host / CUDA batches, stream chunks and two workers on one card give the same frames; unset, the node is the
package's own generator exactly as before."""
import importlib

import pytest
import torch

from helpers import natural_frames

pytestmark = pytest.mark.gpu

I, SAT = 0.3, 0.4
BURN = ((1001,), (7, 13), (3, 5, 3))                       # odd draws that move the offset before each case


def _gen():
    return torch.cuda.default_generators[0]


def _burn(seed):
    torch.cuda.manual_seed(seed)
    for shape in BURN:
        torch.randn(shape, device="cuda")
    return _gen().get_offset()


def _node(pkg, monkeypatch, x, batch_size, intensity=I, sat=SAT):
    monkeypatch.setenv("VRGDG_GRAIN_NOISE", "torch_cuda")
    return pkg.NODE_CLASS_MAPPINGS["FastFilmGrain"]().apply_grain(x, intensity, sat, batch_size)[0]


def _reference_draws(x, batch_size):
    """the reference's noise: torch.randn_like per mini-batch, in the frame dtype"""
    step = batch_size if batch_size > 0 else x.shape[0]
    return torch.cat([torch.randn_like(x[i:i + step]) for i in range(0, x.shape[0], step)])


def _within_one_spacing(a, b):
    ia, ib = a.view(torch.int16).to(torch.int32), b.view(torch.int16).to(torch.int32)
    return bool(((a == b) | ((ia - ib).abs() <= 1)).all())


def _check(pkg, oracle, monkeypatch, x, batch_size, offset):
    """node vs reference from the same generator state: frames and the offset afterwards"""
    gen = _gen()
    gen.set_offset(offset)
    if x.dtype == torch.float32:
        want = oracle.film_grain(x, I, SAT, batch_size)
    else:
        # the project's 16-bit rule: the oracle on the up-cast input with the reference's 16-bit draws, rounded once
        z = _reference_draws(x, batch_size).float()
        want = (x.float() + oracle.grain_mix(z, SAT) * I).clamp(0.0, 1.0).to(x.dtype)
    after = gen.get_offset()
    gen.set_offset(offset)
    got = _node(pkg, monkeypatch, x, batch_size)
    assert gen.get_offset() == after
    assert got.device == x.device and got.dtype == x.dtype
    if x.dtype == torch.float32:
        assert torch.equal(got, want)
    else:
        assert _within_one_spacing(got, want)
    return got


@pytest.mark.parametrize("batch_size", [0, 1, 3, 4])
@pytest.mark.parametrize("shape", [(17, 23), (1080, 1920)], ids=lambda s: "%dx%d" % s)
def test_node_matches_the_reference_on_cuda(pkg, oracle, monkeypatch, cuda_device, shape, batch_size):
    x = natural_frames(7, *shape, seed=1).cuda()
    _check(pkg, oracle, monkeypatch, x, batch_size, _burn(11))


@pytest.mark.parametrize("batch_size", [0, 3])
def test_node_matches_the_reference_on_a_4k_frame_group(pkg, oracle, monkeypatch, cuda_device, batch_size):
    x = natural_frames(7, 2160, 3840, seed=2).cuda()
    _check(pkg, oracle, monkeypatch, x, batch_size, _burn(12))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=str)
@pytest.mark.parametrize("shape", [(17, 23), (1080, 1920)], ids=lambda s: "%dx%d" % s)
def test_16bit_frames_within_one_spacing(pkg, oracle, monkeypatch, cuda_device, shape, dtype):
    x = natural_frames(7, *shape, seed=3).to("cuda", dtype)
    for batch_size in (0, 3):
        _check(pkg, oracle, monkeypatch, x, batch_size, _burn(13))


@pytest.mark.parametrize("offset", [4 * (2**32 - 5), 2**34 + 12], ids=["carry_mid_draw", "past_2^34"])
def test_offsets_that_carry_into_the_second_counter_word(pkg, oracle, monkeypatch, cuda_device, offset):
    x = natural_frames(7, 1080, 1920, seed=4).cuda()
    _burn(14)
    for batch_size in (3, 0):
        _check(pkg, oracle, monkeypatch, x, batch_size, offset)


def test_consecutive_calls_continue_the_stream(pkg, oracle, monkeypatch, cuda_device):
    x = natural_frames(5, 45, 67, seed=5).cuda()
    y = natural_frames(3, 64, 48, seed=6).cuda()
    o0 = _burn(15)
    want = [oracle.film_grain(x, I, SAT, 2), oracle.film_grain(y, I, SAT, 4)]
    after = _gen().get_offset()
    _gen().set_offset(o0)
    got = [_node(pkg, monkeypatch, x, 2), _node(pkg, monkeypatch, y, 4)]
    assert _gen().get_offset() == after
    assert all(torch.equal(g, w) for g, w in zip(got, want))


def test_host_chunks_and_two_workers_equal_the_cuda_batch(pkg, monkeypatch, cuda_device):
    x = natural_frames(7, 40, 56, seed=7)
    mod = importlib.import_module(pkg.__name__ + ".filter_nodes")
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    o0 = _burn(16)
    want = _node(pkg, monkeypatch, x.cuda(), 3).cpu()
    after = _gen().get_offset()
    runs = {}
    _gen().set_offset(o0)
    runs["host"] = _node(pkg, monkeypatch, x, 3)
    monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(40 * 56 * 3 * 4))          # one frame per upload chunk
    _gen().set_offset(o0)
    runs["chunks"] = _node(pkg, monkeypatch, x, 3)
    monkeypatch.delenv("VRGDG_STREAM_CHUNK_BYTES")
    monkeypatch.setattr(mod, "devices_from_env", lambda: [torch.device("cuda", 0), torch.device("cuda", 0)])
    _gen().set_offset(o0)
    runs["two_workers"] = _node(pkg, monkeypatch, x, 3)
    for name, got in runs.items():
        assert got.device.type == "cpu" and torch.equal(got, want), name
    assert _gen().get_offset() == after


def test_unset_keeps_the_package_generator(pkg, monkeypatch, cuda_device):
    """unset or "vrgdg": one seed from the CPU generator and the PER_CLIP kernel, as before; the CUDA generator is not touched"""
    nv, ops = pkg._native, pkg.ops
    mod = importlib.import_module(pkg.__name__ + ".filter_nodes")
    node = pkg.NODE_CLASS_MAPPINGS["FastFilmGrain"]()
    x = natural_frames(5, 33, 47, seed=8).cuda()
    o0 = _burn(17)
    for raw in (None, "vrgdg"):
        if raw is None:
            monkeypatch.delenv("VRGDG_GRAIN_NOISE", raising=False)
        else:
            monkeypatch.setenv("VRGDG_GRAIN_NOISE", raw)
        torch.random.default_generator.manual_seed(99)             # the CPU generator alone (torch.manual_seed reseeds CUDA too)
        got = node.apply_grain(x, I, SAT, 2)[0]
        torch.random.default_generator.manual_seed(99)
        want = ops.grain(x, I, SAT, 1.0 - SAT, mod.draw_seed(), frame0=0, seed_mode=nv.SEED_PER_CLIP)
        assert torch.equal(got, want)
        assert _gen().get_offset() == o0
    _gen().set_offset(o0)
    assert not torch.equal(got, _node(pkg, monkeypatch, x, 2))

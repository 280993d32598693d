"""VRGDG_B200_PostChain with VRGDG_GRAIN_NOISE=torch_cuda on the GPU: the noise kernel equals the reference's torch.randn_like
mini-batch draws, the node's grain equals FastFilmGrain's in that mode, the whole chain equals the four stock nodes run one after
the other in that mode, and the global generator is left where those nodes leave it; host / CUDA batches, stream chunks and two
workers on one card give the same frames; unset, the node is the package's own generator exactly as before."""
import importlib
import os

import pytest
import torch

import chain_matrix as cmx
from helpers import LUTS, natural_frames

pytestmark = pytest.mark.gpu

I, SAT = 0.3, 0.4
LUT_NAME = "B200 Vintage 33.cube"
BURN = ((1001,), (7, 13), (3, 5, 3))                       # odd draws that move the offset before each case


def _gen():
    return torch.cuda.default_generators[0]


def _burn(seed):
    torch.cuda.manual_seed(seed)
    for shape in BURN:
        torch.randn(shape, device="cuda")
    return _gen().get_offset()


def _reference_draws(x, batch_size):
    """the reference's noise: torch.randn_like per mini-batch, in the frame dtype"""
    step = batch_size if batch_size > 0 else x.shape[0]
    return torch.cat([torch.randn_like(x[i:i + step]) for i in range(0, x.shape[0], step)])


def _chain_node(pkg, monkeypatch, x, batch_size, match=None, lut=None, sharpen="none", raw="torch_cuda"):
    if raw is None:
        monkeypatch.delenv("VRGDG_GRAIN_NOISE", raising=False)
    else:
        monkeypatch.setenv("VRGDG_GRAIN_NOISE", raw)
    node = pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_PostChain"]()
    return node.apply_chain(x, I, SAT, 0.7, lut or "none", 6.0, sharpen, 0.5, False, batch_size, reference_image=match)[0]


def _stock_nodes(pkg, monkeypatch, x, batch_size, match=None, lut=None, sharpen="none"):
    """FastFilmGrain -> ColorMatchToReference -> VRGDG_LUTS -> FastUnsharpSharpen, grain drawn under torch_cuda"""
    monkeypatch.setenv("VRGDG_GRAIN_NOISE", "torch_cuda")
    y = pkg.NODE_CLASS_MAPPINGS["FastFilmGrain"]().apply_grain(x, I, SAT, batch_size)[0]
    if match is not None:
        y = pkg.ColorMatchToReference().match_color(y, match, 0.7, 1)[0]
    if lut is not None:
        y = pkg.VRGDG_LUTS().apply_lut(y, lut, "auto", 6.0)[0]
    if sharpen == "unsharp":
        y = pkg.FastUnsharpSharpen().apply_unsharp(y, 0.5, False)[0]
    return y


def _both(pkg, monkeypatch, x, batch_size, offset, **kw):
    """(node, stock nodes) from the same generator state; the offsets after them must agree"""
    gen = _gen()
    gen.set_offset(offset)
    want = _stock_nodes(pkg, monkeypatch, x, batch_size, **kw)
    after = gen.get_offset()
    gen.set_offset(offset)
    got = _chain_node(pkg, monkeypatch, x, batch_size, **kw)
    assert gen.get_offset() == after
    assert got.device == x.device and got.dtype == x.dtype
    return got, want


# ---- the noise kernel ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16], ids=str)
@pytest.mark.parametrize("batch_size", [0, 1, 3, 4])
@pytest.mark.parametrize("shape", [(17, 23), (1080, 1920)], ids=lambda s: "%dx%d" % s)
def test_noise_kernel_equals_the_reference_draws(pkg, cuda_device, shape, batch_size, dtype):
    """every window of the clip, whole or starting and ending mid-draw, is the matching slice of the reference's draws"""
    x = torch.zeros((7,) + shape + (3,), device="cuda", dtype=dtype)
    o0 = _burn(21)
    want = _reference_draws(x, batch_size)
    seed, step = _gen().initial_seed(), batch_size if batch_size > 0 else 7
    for f0, k in ((0, 7), (2, 3), (5, 2), (1, 1)):
        got = pkg.ops.grain_noise_torch_global(x[f0:f0 + k], seed, o0, f0, 7, step)
        assert got.dtype == dtype and got.shape == x[f0:f0 + k].shape
        assert torch.equal(got, want[f0:f0 + k]), (f0, k)


@pytest.mark.parametrize("offset", [4 * (2**32 - 5), 2**34 + 12], ids=["carry_mid_draw", "past_2^34"])
def test_noise_kernel_at_offsets_that_carry_into_the_second_counter_word(pkg, cuda_device, offset):
    x = torch.zeros(7, 1080, 1920, 3, device="cuda")
    _burn(22)
    seed = _gen().initial_seed()
    for batch_size in (3, 0):
        _gen().set_offset(offset)
        want = _reference_draws(x, batch_size)
        step = batch_size if batch_size > 0 else 7
        assert torch.equal(pkg.ops.grain_noise_torch_global(x, seed, offset, 0, 7, step), want)
        assert torch.equal(pkg.ops.grain_noise_torch_global(x[4:6], seed, offset, 4, 7, step), want[4:6])


# ---- the node -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch_size", [0, 1, 3, 4])
def test_grain_only_node_equals_film_grain(pkg, monkeypatch, cuda_device, batch_size):
    x = natural_frames(7, 45, 67, seed=1).cuda()
    got, want = _both(pkg, monkeypatch, x, batch_size, _burn(23))
    assert torch.equal(got, want)


@pytest.mark.parametrize("shape", [(17, 23), (1080, 1920)], ids=lambda s: "%dx%d" % s)
def test_chain_equals_the_four_stock_nodes(pkg, monkeypatch, cuda_device, shape):
    """grain -> 33^3 LUT -> unsharp exactly; with colour match within the bar of the default mode's comparison"""
    x = natural_frames(5, *shape, seed=2).cuda()
    ref = (natural_frames(1, 50, 60, seed=3) * 0.8).cuda()
    for batch_size in (0, 2):
        got, want = _both(pkg, monkeypatch, x, batch_size, _burn(24), lut=LUT_NAME, sharpen="unsharp")
        assert torch.equal(got, want)
        got, want = _both(pkg, monkeypatch, x, batch_size, _burn(25), match=ref, lut=LUT_NAME, sharpen="unsharp")
        assert float((got - want).abs().max()) <= 2e-6


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=str)
@pytest.mark.parametrize("cm", [False, True], ids=["no_cm", "cm"])
def test_16bit_chain_against_the_oracle_on_the_reference_draws(pkg, oracle, monkeypatch, cuda_device, dtype, cm):
    """the oracle composition on the up-cast input with the reference's 16-bit draws, within the chain matrix's bar for the
    external-noise case"""
    x = natural_frames(5, 72, 176, seed=4).to("cuda", dtype)
    ref = natural_frames(1, 50, 60, seed=5) * 0.8
    o0 = _burn(26)
    z = _reference_draws(x, 2).float().cpu()
    after = _gen().get_offset()
    _gen().set_offset(o0)
    got = _chain_node(pkg, monkeypatch, x, 2, match=ref.to("cuda", dtype) if cm else None, lut=LUT_NAME, sharpen="unsharp")
    assert _gen().get_offset() == after
    want = oracle.chain_compose(x.cpu(), grain=dict(intensity=I, saturation_mix=SAT),
                                colormatch=dict(reference_image=ref.to(dtype).float(), strength=0.7) if cm else None,
                                lut=dict(lut_data=oracle.parse_cube(os.path.join(LUTS, LUT_NAME)), strength=6.0),
                                stencil=dict(op=1, border=0, strength=0.5), z=z)
    bar = cmx.ULP["f16" if dtype == torch.float16 else "bf16"] + (cmx.BAR_CM if cm else 0.0)
    assert float((got.cpu().float() - want.float()).abs().max()) <= bar


def test_consecutive_calls_continue_the_stream(pkg, monkeypatch, cuda_device):
    x = natural_frames(5, 45, 67, seed=6).cuda()
    y = natural_frames(3, 64, 48, seed=7).cuda()
    o0 = _burn(27)
    want = [_stock_nodes(pkg, monkeypatch, x, 2, lut=LUT_NAME), _stock_nodes(pkg, monkeypatch, y, 4, lut=LUT_NAME)]
    after = _gen().get_offset()
    _gen().set_offset(o0)
    got = [_chain_node(pkg, monkeypatch, x, 2, lut=LUT_NAME), _chain_node(pkg, monkeypatch, y, 4, lut=LUT_NAME)]
    assert _gen().get_offset() == after
    assert all(torch.equal(g, w) for g, w in zip(got, want))


def test_host_chunks_and_two_workers_equal_the_cuda_batch(pkg, monkeypatch, cuda_device):
    x = natural_frames(7, 40, 56, seed=8)
    ref = natural_frames(1, 30, 40, seed=9) * 0.8
    mod = importlib.import_module(pkg.__name__ + ".chain_nodes")
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    kw = dict(match=ref, lut=LUT_NAME, sharpen="unsharp")
    o0 = _burn(28)
    want = _chain_node(pkg, monkeypatch, x.cuda(), 3, **kw).cpu()
    after = _gen().get_offset()
    runs = {}
    _gen().set_offset(o0)
    runs["host"] = _chain_node(pkg, monkeypatch, x, 3, **kw)
    monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(40 * 56 * 3 * 4))          # one frame per upload chunk
    _gen().set_offset(o0)
    runs["chunks"] = _chain_node(pkg, monkeypatch, x, 3, **kw)
    monkeypatch.delenv("VRGDG_STREAM_CHUNK_BYTES")
    monkeypatch.setattr(mod, "devices_from_env", lambda: [torch.device("cuda", 0), torch.device("cuda", 0)])
    _gen().set_offset(o0)
    runs["two_workers"] = _chain_node(pkg, monkeypatch, x, 3, **kw)
    for name, got in runs.items():
        assert got.device.type == "cpu" and torch.equal(got, want), name
    assert _gen().get_offset() == after


def test_device_batch_in_noise_sub_batches_equals_one_call(pkg, monkeypatch, cuda_device):
    """a CUDA batch larger than one pipeline chunk makes its noise one chunk at a time; the frames do not change"""
    x = natural_frames(7, 40, 56, seed=10).cuda()
    ref = (natural_frames(1, 30, 40, seed=11) * 0.8).cuda()
    o0 = _burn(29)
    want = _chain_node(pkg, monkeypatch, x, 0, match=ref, lut=LUT_NAME, sharpen="unsharp")
    after = _gen().get_offset()
    monkeypatch.setenv("VRGDG_STREAM_CHUNK_BYTES", str(2 * 40 * 56 * 3 * 4))      # two frames of noise at a time
    _gen().set_offset(o0)
    got = _chain_node(pkg, monkeypatch, x, 0, match=ref, lut=LUT_NAME, sharpen="unsharp")
    assert torch.equal(got, want) and _gen().get_offset() == after


def test_4k_group_with_colour_match_on_the_fplane_schedule(pkg, monkeypatch, cuda_device):
    """fp32 4K frames (W % 4 == 0) take vrgdg_chain_cm_apply's f-plane schedule, in groups of frames"""
    x = natural_frames(3, 2160, 3840, seed=12).cuda()
    ref = (natural_frames(1, 120, 200, seed=13) * 0.8).cuda()
    got, want = _both(pkg, monkeypatch, x, 2, _burn(30), match=ref, lut=LUT_NAME, sharpen="unsharp")
    assert float((got - want).abs().max()) <= 2e-6


def test_unset_keeps_the_package_generator(pkg, monkeypatch, cuda_device):
    """unset or "vrgdg": one seed from the CPU generator and the in-kernel generator, as before; the CUDA generator is not touched"""
    nv = pkg._native
    fn = importlib.import_module(pkg.__name__ + ".filter_nodes")
    x = natural_frames(5, 33, 47, seed=14).cuda()
    lut = pkg.VRGDG_LUTS._load_lut(LUT_NAME)
    o0 = _burn(31)
    for raw in (None, "vrgdg"):
        torch.random.default_generator.manual_seed(99)             # the CPU generator alone (torch.manual_seed reseeds CUDA too)
        got = _chain_node(pkg, monkeypatch, x, 2, lut=LUT_NAME, sharpen="unsharp", raw=raw)
        torch.random.default_generator.manual_seed(99)
        chain = pkg.chain.PostChain(grain=dict(intensity=I, saturation_mix=SAT, seed=fn.draw_seed()), lut=dict(lut_data=lut, strength=6.0),
                                    stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5, border=nv.BORDER_REPLICATE), device=x.device)
        assert torch.equal(got, chain(x))
        assert _gen().get_offset() == o0
    _gen().set_offset(o0)
    assert not torch.equal(got, _chain_node(pkg, monkeypatch, x, 2, lut=LUT_NAME, sharpen="unsharp"))

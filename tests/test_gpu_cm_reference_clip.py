"""Colour match against a reference clip on the GPU.  vrgdg_chain_cm_apply_refs is torch.equal to today's two steps
(vrgdg_lab_moments over the whole reference clip, then vrgdg_chain_cm_apply with n_ref = B) on every dtype, grain mode, stage set,
schedule, group size and reference size; ColorMatchToReference with n_ref == B equals that computation whatever the chunks, workers
and devices; VRGDG_B200_PostChain with a reference clip equals PostChain on precomputed per-frame sums, the four stock nodes under
VRGDG_GRAIN_NOISE=torch_cuda within the colour-match bar, and the oracle frame by frame; and the reference clip no longer has to fit
on the card next to the frames."""
import importlib
import os

import pytest
import torch

from helpers import LUTS, natural_frames

pytestmark = pytest.mark.gpu

LUT_NAME = "B200 Vintage 33.cube"
CM_T, LUT_BLEND = 0.8, 0.6
GRAIN = dict(intensity=0.04, saturation_mix=0.5)
DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
# grain off, the in-kernel generator, external noise in exact and in fast arithmetic
GRAINS = ("off", "gen", "ext", "ext_fast")
SCHEDULES = (dict(), dict(serial=True), dict(recompute=True))      # default = pipelined for fp32 + LUT over several groups


def _desc(pkg, dev, grain, lut, unsharp, keep):
    nv = pkg._native
    d = nv.ChainDesc()
    d.colormatch_enabled, d.cm_t, d.cm_one_minus_t = 1, CM_T, 1.0 - CM_T
    if grain != "off":
        s = GRAIN["saturation_mix"]
        d.grain_enabled, d.grain_intensity, d.grain_sat, d.grain_one_minus_sat = 1, GRAIN["intensity"], s, 1.0 - s
        d.grain_seed, d.grain_frame0, d.grain_seed_mode = 0x5EED, 9, nv.SEED_PER_FRAME
    if lut:
        data = pkg.VRGDG_LUTS._parse_cube_file(os.path.join(LUTS, LUT_NAME))
        packed = pkg.ops.pack_lut(data["lut"], dev)
        keep.append(packed)
        dmin = data["domain_min"].float()
        span = torch.clamp(data["domain_max"].float() - dmin, min=1e-6)
        d.lut_enabled, d.lut, d.lut_size = 1, packed.data.data_ptr(), packed.size
        d.lut_dmin, d.lut_dspan = (type(d.lut_dmin))(*dmin.tolist()), (type(d.lut_dspan))(*span.tolist())
        d.lut_blend, d.lut_one_minus_blend = LUT_BLEND, 1.0 - LUT_BLEND
    if unsharp:
        d.stencil_op, d.stencil_strength, d.stencil_border = nv.STENCIL_BOX_UNSHARP, 0.5, nv.BORDER_REPLICATE
    return d


def _both_library_paths(pkg, x, refs, d, z, fast, group, sched):
    got, _ = pkg.ops.chain_cm_apply_refs(x, d, refs, ext_noise=z, fast_math=fast, group_frames=group, **sched)
    want, _ = pkg.ops.chain_cm_apply(x, d, pkg.ops.lab_moments(refs), ext_noise=z, fast_math=fast, group_frames=group, **sched)
    return got, want


# ---- library ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stages", ["cm", "cm_lut", "cm_lut_unsharp"])
@pytest.mark.parametrize("dtype", list(DT))
def test_entry_equals_whole_clip_moments_then_one_call(pkg, cuda_device, dtype, stages):
    """B = 7 frames (not a multiple of 3), groups of 1, 3 and the default; references at the frames' size and at another size"""
    x = natural_frames(7, 72, 96, seed=1).to(cuda_device, DT[dtype])
    z = torch.randn(x.shape, generator=torch.Generator().manual_seed(2)).to(cuda_device, DT[dtype])
    refs_by_size = {"same": (natural_frames(7, 72, 96, seed=3) * 0.8 + 0.1).to(cuda_device, DT[dtype]),
                    "other": (natural_frames(7, 36, 52, seed=4) * 0.7 + 0.2).to(cuda_device, DT[dtype])}
    for grain in GRAINS:
        keep = []
        d = _desc(pkg, cuda_device, grain, "lut" in stages, "unsharp" in stages, keep)
        noise = z if grain.startswith("ext") else None
        for size, refs in refs_by_size.items():
            for sched in SCHEDULES:
                for group in (1, 3, 0):
                    got, want = _both_library_paths(pkg, x, refs, d, noise, grain == "ext_fast", group, sched)
                    assert torch.equal(got, want), (grain, size, sched, group)


def test_entry_on_a_4k_group_of_the_fplane_schedule(pkg, cuda_device):
    """two fp32 4K frames form one group that stores f-planes; 4K and 1080p reference clips, grain from the generator"""
    x = natural_frames(2, 2160, 3840, seed=5).to(cuda_device)
    keep = []
    d = _desc(pkg, cuda_device, "gen", True, True, keep)
    for refs in (natural_frames(2, 2160, 3840, seed=6).to(cuda_device) * 0.8, natural_frames(2, 1080, 1920, seed=7).to(cuda_device) * 0.9):
        got, want = _both_library_paths(pkg, x, refs, d, None, False, 0, {})
        assert torch.equal(got, want)


def test_entry_960x540_references_for_1080p_frames_in_pipelined_groups(pkg, cuda_device):
    x = natural_frames(5, 1080, 1920, seed=8).to(cuda_device)
    refs = natural_frames(5, 540, 960, seed=9).to(cuda_device) * 0.85
    keep = []
    d = _desc(pkg, cuda_device, "gen", True, True, keep)
    for group in (2, 0):
        got, want = _both_library_paths(pkg, x, refs, d, None, False, group, {})
        assert torch.equal(got, want), group


# ---- ColorMatchToReference ------------------------------------------------------------------------------------------------------
def _today(pkg, x, refs):
    """today's computation with a reference clip: statistics of the whole clip in the frames' dtype, then one call"""
    nv = pkg._native
    d = nv.ChainDesc()
    d.colormatch_enabled, d.cm_t, d.cm_one_minus_t = 1, CM_T, 1.0 - CM_T
    dev = torch.device("cuda", 0)
    return pkg.ops.chain_cm_apply(x.to(dev), d, pkg.ops.lab_moments(refs.to(dev).to(x.dtype)))[0].cpu()


@pytest.mark.parametrize("dtype", ["f32", "f16"])
def test_colormatch_node_with_a_reference_clip_equals_whole_clip_statistics(pkg, monkeypatch, cuda_device, dtype):
    fn = importlib.import_module(pkg.__name__ + ".filter_nodes")
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    x = natural_frames(7, 40, 56, seed=10).to(DT[dtype])
    refs = natural_frames(7, 30, 44, seed=11) * 0.8                    # fp32 references: converted to the frames' dtype per chunk
    want = _today(pkg, x, refs)
    node = pkg.ColorMatchToReference()
    for chunk in (1, 2, 7):
        for frames_dev in ("cpu", "cuda"):
            for refs_dev in ("cpu", "cuda"):                            # the reference clip on the same and on the other device type
                got = node.match_color(x.to(frames_dev), refs.to(refs_dev), CM_T, chunk)[0]
                assert got.device.type == frames_dev and torch.equal(got.cpu(), want), (chunk, frames_dev, refs_dev)
    monkeypatch.setattr(fn, "devices_from_env", lambda: [torch.device("cuda", 0), torch.device("cuda", 0)])    # two workers, one card
    for chunk in (1, 2):
        got = node.match_color(x, refs, CM_T, chunk)[0]
        assert torch.equal(got, want), chunk


def test_colormatch_node_device_memory_follows_the_chunk_not_the_reference_clip(pkg, monkeypatch, cuda_device):
    """24 host 1080p fp32 frames against 24 host reference frames (597 MB) in chunks of 4: the reference clip adds at most two chunks
    of reference frames to the device peak of the same call with one reference frame (the frames' own pipeline slots, result and
    f-plane scratch), where today's path added the whole clip"""
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    x = torch.rand(24, 1080, 1920, 3, generator=torch.Generator().manual_seed(12))
    refs = torch.rand(24, 1080, 1920, 3, generator=torch.Generator().manual_seed(13)) * 0.8
    clip_bytes = refs.numel() * refs.element_size()
    chunk_bytes = 4 * refs[0].numel() * refs.element_size()
    node = pkg.ColorMatchToReference()
    peaks = {}
    for name, r in (("one", refs[:1]), ("clip", refs)):
        node.match_color(x[:8], r[:8] if len(r) > 1 else r, CM_T, 4)    # warm-up: kernels loaded, pinned staging buffers cached
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        got = node.match_color(x, r, CM_T, 4)[0]
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
    print("device peak: one reference %.1f MB, reference clip %.1f MB (clip %.1f MB)" % (peaks["one"] / 1e6, peaks["clip"] / 1e6, clip_bytes / 1e6))
    assert peaks["clip"] - peaks["one"] <= 2 * chunk_bytes
    assert peaks["clip"] < peaks["one"] + clip_bytes / 2
    assert torch.equal(got[20:], _today(pkg, x[20:], refs[20:]))


# ---- the Post Chain ------------------------------------------------------------------------------------------------------------
def _post_node(pkg, x, refs, batch_size, grain=0.04, lut=LUT_NAME, sharpen="unsharp"):
    return pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_PostChain"]().apply_chain(x, grain, 0.5, CM_T, lut or "none", 6.0, sharpen, 0.5, False,
                                                                          batch_size, reference_image=refs)[0]


def test_postchain_node_with_a_reference_clip_equals_postchain_on_per_frame_sums(pkg, monkeypatch, cuda_device):
    """same chain, same seed: the node's streamed reference clip against PostChain driven with ref_sums [B,7], whole batch and chunked"""
    nv = pkg._native
    fn = importlib.import_module(pkg.__name__ + ".filter_nodes")
    monkeypatch.delenv("VRGDG_GRAIN_NOISE", raising=False)
    monkeypatch.delenv("VRGDG_DEVICES", raising=False)
    x = natural_frames(7, 48, 64, seed=14)
    refs = natural_frames(7, 24, 40, seed=15) * 0.8
    lut = pkg.VRGDG_LUTS._load_lut(LUT_NAME)
    torch.random.default_generator.manual_seed(77)
    seed = fn.draw_seed()
    chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=seed),
                                colormatch=dict(ref_sums=pkg.ops.lab_moments(refs.to(cuda_device)), strength=CM_T),
                                lut=dict(lut_data=lut, strength=6.0),
                                stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5, border=nv.BORDER_REPLICATE), device=cuda_device)
    want = chain(x.to(cuda_device)).cpu()
    assert torch.equal(chain.run_host(x, chunk_frames=3), want)            # per-frame sums sliced by the absolute frame index
    for frames_dev in ("cpu", "cuda"):
        for batch_size in (0, 3):
            torch.random.default_generator.manual_seed(77)
            got = _post_node(pkg, x.to(frames_dev), refs, batch_size)
            assert torch.equal(got.cpu(), want), (frames_dev, batch_size)
    # PostChain with reference_frames: the fused call, the three-call path, timing, run_host on two workers of one card
    clip = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=seed), colormatch=dict(reference_frames=refs, strength=CM_T),
                               lut=dict(lut_data=lut, strength=6.0),
                               stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5, border=nv.BORDER_REPLICATE), device=cuda_device)
    assert torch.equal(clip(x.to(cuda_device)).cpu(), want)
    assert torch.equal(clip(x[2:6].to(cuda_device), first_frame=2).cpu(), want[2:6])
    clip.split = True
    split = clip(x.to(cuda_device)).cpu()
    clip.split, clip.timing = False, []
    timed = clip(x[3:].to(cuda_device), first_frame=3).cpu()
    clip.timing = None
    assert float((split - want).abs().max()) <= 2e-6 and torch.equal(timed, split[3:])
    two = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=seed), colormatch=dict(reference_frames=refs.to(cuda_device),
                              strength=CM_T), lut=dict(lut_data=lut, strength=6.0),
                              stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5, border=nv.BORDER_REPLICATE), devices=[cuda_device, cuda_device])
    assert torch.equal(two.run_host(x, chunk_frames=2), want)


def test_postchain_node_with_a_reference_clip_equals_the_four_stock_nodes_under_torch_cuda(pkg, monkeypatch, cuda_device):
    """FastFilmGrain -> ColorMatchToReference(reference clip) -> VRGDG_LUTS -> FastUnsharpSharpen, grain from the global generator"""
    monkeypatch.setenv("VRGDG_GRAIN_NOISE", "torch_cuda")
    gen = torch.cuda.default_generators[0]
    x = natural_frames(5, 45, 64, seed=16).to(cuda_device)
    refs = (natural_frames(5, 30, 40, seed=17) * 0.8).to(cuda_device)
    for batch_size in (0, 2):
        torch.cuda.manual_seed(31)
        o0 = gen.get_offset()
        y = pkg.NODE_CLASS_MAPPINGS["FastFilmGrain"]().apply_grain(x, 0.3, 0.5, batch_size)[0]
        y = pkg.ColorMatchToReference().match_color(y, refs, CM_T, 1)[0]
        y = pkg.VRGDG_LUTS().apply_lut(y, LUT_NAME, "auto", 6.0)[0]
        want = pkg.FastUnsharpSharpen().apply_unsharp(y, 0.5, False)[0]
        after = gen.get_offset()
        gen.set_offset(o0)
        got = _post_node(pkg, x, refs, batch_size, grain=0.3)
        assert gen.get_offset() == after
        assert float((got - want).abs().max()) <= 2e-6, batch_size


def test_postchain_node_pairs_each_frame_with_its_own_reference(pkg, oracle, monkeypatch, cuda_device):
    monkeypatch.delenv("VRGDG_GRAIN_NOISE", raising=False)
    x = natural_frames(5, 40, 56, seed=18)
    refs = torch.stack([(natural_frames(1, 32, 48, seed=19 + i)[0] * (0.5 + 0.1 * i)).clamp(0, 1) for i in range(5)])
    got = _post_node(pkg, x, refs, 2, grain=0.0, lut=None, sharpen="none")
    for i in range(5):
        want = oracle.color_match(x[i:i + 1], refs[i:i + 1], CM_T, 1)
        assert float((got[i:i + 1] - want).abs().max()) <= 1e-5, i

"""Every stage combination of the fused chain against the oracle composition (oracle.chain_compose), not against other kernels.

The matrix (tests/chain_matrix.py): every subset of {grain, colour match, LUT, post grain} x {no stencil, unsharp-replicate}, and
every (op, border) pair the reference owns behind grain + LUT and behind grain + colour match + LUT; fp32, fp16, bf16 and uint8 BGR
frames; external noise in exact and fast arithmetic and the in-kernel generator in both seed modes (non-zero first frame; post
grain always draws from the generator with its own seed); every colour-match schedule; a multi-tile TMA shape, a ragged shape on the
generic loader and the TMA shape under VRGDG_NO_TMA=1.  (op, border) pairs without a reference function (a NumPy-path op with zero
borders, a torch-path op with replicated borders) are outside the matrix.  Error bars: chain_matrix.float_bar / half_bar."""
import functools
import os

import pytest
import torch

import chain_matrix as cmx
from helpers import LUTS, natural_frames

pytestmark = pytest.mark.gpu

DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16, "u8": torch.uint8}
LUT_FILE = os.path.join(LUTS, "B200 Vintage 33.cube")
GRAIN = dict(intensity=0.04, saturation_mix=0.5)
POST = dict(intensity=0.03, saturation_mix=0.7)
GRAIN_SEED, POST_SEED, FRAME0 = 0x1234_5678_9ABC, 977, 11
CM_STRENGTH, LUT_STRENGTH = 0.8, 8.0
SEED_MODE = {"clip": 0, "frame": 1}


def post_seed_mode(c):
    """both post-grain seed modes occur; a per-frame post stage behind a per-frame first stage would share its Philox key"""
    return SEED_MODE["clip"] if c.noise == "frame" else SEED_MODE["frame"]


@pytest.fixture(scope="module")
def env(pkg, oracle, cuda_device):
    ref = (natural_frames(1, 50, 60, seed=99) * 0.8 + 0.1).clamp(0, 1)
    return dict(lut=pkg.VRGDG_LUTS._parse_cube_file(LUT_FILE), olut=oracle.parse_cube(LUT_FILE), ref=ref,
                ref_sums=pkg.ops.lab_moments(ref.to(cuda_device)))


@functools.lru_cache(maxsize=None)
def _frames(dtype, shape):
    B, H, W = cmx.SHAPES[shape]
    x = natural_frames(B, H, W, seed=B * 100000 + H * 1000 + W)
    return (x * 255).round().clamp(0, 255).to(torch.uint8) if dtype == "u8" else x.to(DT[dtype])


@functools.lru_cache(maxsize=None)
def _ext_noise(dtype, shape):
    B, H, W = cmx.SHAPES[shape]
    z = torch.randn(B, H, W, 3, generator=torch.Generator().manual_seed(B * 7 + H * 3 + W))
    return z if dtype in ("f32", "u8") else z.to(DT[dtype])        # frame dtype; float32 for byte frames


@functools.lru_cache(maxsize=None)
def _gen_noise(pkg, seed, mode, shape):
    B, H, W = cmx.SHAPES[shape]
    return pkg.ops.grain_noise(B, H, W, seed, FRAME0, mode, device="cuda").cpu()


def _oracle_key(c):
    shape = "tma" if c.shape == "notma" else c.shape      # same frames, same result
    return c._replace(schedule="default", shape=shape)


_ORACLE = {}


def _expected(pkg, oracle, env, c):
    key = _oracle_key(c)
    if key not in _ORACLE:
        z = None
        if c.grain:
            z = _ext_noise(c.dtype, key.shape).float() if c.noise.startswith("ext") else _gen_noise(pkg, GRAIN_SEED, SEED_MODE[c.noise], key.shape)
        post_z = _gen_noise(pkg, POST_SEED, post_seed_mode(c), key.shape) if c.post else None
        st = None
        if c.stencil:
            st = dict(op=c.stencil[0], border=c.stencil[1], strength=cmx.STENCIL_STRENGTH[c.stencil[0]])
        _ORACLE[key] = oracle.chain_compose(_frames(c.dtype, key.shape), grain=GRAIN if c.grain else None,
                                            colormatch=dict(reference_image=env["ref"], strength=CM_STRENGTH) if c.cm else None,
                                            lut=dict(lut_data=env["olut"], strength=LUT_STRENGTH) if c.lut else None, stencil=st,
                                            post_grain=POST if c.post else None, z=z, post_z=post_z)
    return _ORACLE[key]


def _run(pkg, env, c, dev):
    nv = pkg._native
    grain = dict(GRAIN, seed=GRAIN_SEED, seed_mode=SEED_MODE.get(c.noise, 0)) if c.grain else None
    chain = pkg.chain.PostChain(grain=grain,
                                colormatch=dict(ref_sums=env["ref_sums"], strength=CM_STRENGTH) if c.cm else None,
                                lut=dict(lut_data=env["lut"], strength=LUT_STRENGTH) if c.lut else None,
                                stencil=dict(op=c.stencil[0], strength=cmx.STENCIL_STRENGTH[c.stencil[0]], border=c.stencil[1]) if c.stencil else None,
                                post_grain=dict(POST, seed=POST_SEED, seed_mode=post_seed_mode(c)) if c.post else None, device=dev)
    chain.split = c.schedule == "split"
    chain.recompute = c.schedule == "recompute"
    chain.serial = c.schedule == "serial"
    chain.group_frames = {"serial": 2, "g1": 1, "g2": 2}.get(c.schedule, 0)
    x = _frames(c.dtype, c.shape).to(dev)
    z = _ext_noise(c.dtype, c.shape).to(dev) if (c.grain and c.noise.startswith("ext")) else None
    if c.shape == "notma":
        os.environ["VRGDG_NO_TMA"] = "1"
    try:
        out = chain(x, first_frame=FRAME0, ext_noise=z, fast_math=c.noise == "ext_fast")
        torch.cuda.synchronize()
        path = nv.last_tile_path()
    finally:
        os.environ.pop("VRGDG_NO_TMA", None)
    return x, out, path


@pytest.mark.parametrize("c", cmx.CASES, ids=cmx.case_id)
def test_chain_matrix_vs_oracle(pkg, oracle, cuda_device, env, c):
    x, out, path = _run(pkg, env, c, cuda_device)
    assert out.dtype == x.dtype and out.shape == x.shape and out.device == x.device
    if c.stencil or c.post:
        want_path = "tma" if c.shape in ("tma", "groups") else "generic"
        assert path == want_path, (path, want_path)
    assert not torch.equal(out, x), "an enabled stage left the frames unchanged"
    want = _expected(pkg, oracle, env, c)
    got = out.cpu()
    if c.dtype == "u8":
        d = (got.int() - want.int()).abs()
        if cmx.float_bar(c) == 0:
            assert torch.equal(got, want), "bytes differ: %d of %d, max %d" % (int((d > 0).sum()), d.numel(), int(d.max()))
        else:
            frac = float((d > 0).double().mean())
            assert int(d.max()) <= 1 and frac < cmx.U8_FLIP_FRACTION, (int(d.max()), frac)
        return
    err = float((got.double() - want.double()).abs().max())
    if c.dtype == "f32":
        bar = cmx.float_bar(c)
        if bar == 0:
            assert torch.equal(got, want), "max |diff| %.3g, want bit-identical" % err
        else:
            assert err <= bar, (err, bar)
    else:
        bar = cmx.half_bar(c)
        assert err <= bar, (err, bar)

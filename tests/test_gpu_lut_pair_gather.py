"""The tile kernels' LUT pre-stage splits every cell sector between the two lanes of a lane pair (lut_eval_lane_pair); the streaming
kernel k_point gathers whole sectors per lane.  Both must give the same bits: the fused k_tile chain grain -> LUT -> stencil is compared
with torch.equal against k_point's grain -> LUT followed by the standalone stencil kernel, on fp32 / fp16 / bf16 / uint8 BGR frames,
33^3 / 64^3 / 65^3 tables, blend strengths 1 and 0.6, corner cells (exact arithmetic) and coefficient cells (fast arithmetic), a
ragged TMA shape (partial tiles, so lanes without pixels in the image serve their partners; every tile's pre-stage ends in a
partial warp), the generic loader and an odd width.

The intermediate is kept in fp32: k_tile never rounds the pre-stage result to the frame type, so the two-kernel side runs on the
up-cast frames and rounds (uint8: truncates) once at the end.  The stencil is the torch-path Laplacian, whose arithmetic does not
depend on the exact / fast switch, plus the NumPy-path box unsharp where both sides run it exactly (fp32 and uint8 frames on
exact arithmetic)."""
import functools
import os

import pytest
import torch

from helpers import LUTS, big_lut_table, natural_frames

pytestmark = pytest.mark.gpu

DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16, "u8": torch.uint8}
SHAPES = {"tma": (2, 45, 208), "notma": (2, 45, 208), "odd": (1, 37, 201)}
GRAIN = dict(intensity=0.04, saturation_mix=0.5, seed=0)


@functools.lru_cache(maxsize=None)
def _lut(pkg, size):
    if size == 33:
        return pkg.VRGDG_LUTS._parse_cube_file(os.path.join(LUTS, "B200 Vintage 33.cube"))
    lut = torch.from_numpy(big_lut_table(size)).float().reshape(size, size, size, 3).contiguous()
    return dict(lut=lut, size=size, domain_min=torch.zeros(3), domain_max=torch.ones(3), title="big %d" % size)


@functools.lru_cache(maxsize=None)
def _inputs(dtype, shape):
    B, H, W = SHAPES[shape]
    x = natural_frames(B, H, W, seed=B * 1000 + W)
    x = (x * 255).round().clamp(0, 255).to(torch.uint8) if dtype == "u8" else x.to(DT[dtype])
    z = torch.randn(B, H, W, 3, generator=torch.Generator().manual_seed(H * 7 + W))
    return x, (z if dtype in ("f32", "u8") else z.to(DT[dtype]))


def _stencils(nv, dtype, fast):
    out = [(nv.STENCIL_LAPLACIAN_GPU, nv.BORDER_ZERO, 0.6), (nv.STENCIL_LAPLACIAN_GPU, nv.BORDER_REPLICATE, 0.6)]
    if dtype in ("f32", "u8") and not fast:
        out.append((nv.STENCIL_BOX_UNSHARP, nv.BORDER_REPLICATE, 0.5))
    return out


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("fast", [False, True], ids=["exact", "fast"])
@pytest.mark.parametrize("strength", [10.0, 6.0], ids=["blend1", "blend06"])
@pytest.mark.parametrize("size", [33, 64, 65])
@pytest.mark.parametrize("dtype", sorted(DT))
def test_tile_lane_pair_gather_equals_per_lane_gather(pkg, cuda_device, dtype, size, strength, fast, shape):
    nv = pkg._native
    x, z = _inputs(dtype, shape)
    xd, zd = x.to(cuda_device), z.to(cuda_device)
    lut = dict(lut_data=_lut(pkg, size), strength=strength)
    # the two-kernel side on fp32 RGB frames holding exactly the values the tile kernel computes with
    if dtype == "u8":
        # x / 255 correctly rounded, as the kernels decode bytes (a CUDA tensor divided by a Python scalar is multiplied by 1/255)
        xf = (xd.float() / torch.full(xd.shape, 255.0, device=cuda_device)).flip(-1).contiguous()
    else:
        xf = xd.float()
    pointwise = pkg.chain.PostChain(grain=GRAIN, lut=lut, device=cuda_device)
    mid = pointwise(xf, ext_noise=zd.float(), fast_math=fast)
    assert mid.dtype == torch.float32
    for op, border, s in _stencils(nv, dtype, fast):
        fused_chain = pkg.chain.PostChain(grain=GRAIN, lut=lut, stencil=dict(op=op, strength=s, border=border), device=cuda_device)
        if shape == "notma":
            os.environ["VRGDG_NO_TMA"] = "1"
        try:
            fused = fused_chain(xd, ext_noise=zd, fast_math=fast)
            torch.cuda.synchronize()
            path = nv.last_tile_path()
        finally:
            os.environ.pop("VRGDG_NO_TMA", None)
        assert path == ("tma" if shape == "tma" else "generic"), path
        want = pkg.ops.stencil3x3(mid, op, s, border)
        if dtype == "u8":
            want = (want * 255.0).clamp(0, 255).to(torch.uint8).flip(-1)
        else:
            want = want.to(DT[dtype])
        assert fused.dtype == x.dtype and fused.shape == x.shape
        assert not torch.equal(fused, xd)
        d = (fused.double() - want.double()).abs()
        assert torch.equal(fused, want), "op %d border %d: %d of %d elements differ, max %.3g" % (
            op, border, int((d > 0).sum()), d.numel(), float(d.max()))

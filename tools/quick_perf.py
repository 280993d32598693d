"""Scratch micro-benchmark of every kernel family (GPU box only).  Not the contract bench (bench.py)."""
import importlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
pkg = importlib.import_module("comfyui-vrgamedevgirl_b200")
from helpers import LUTS, natural_frames  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _clocks import Clocks  # noqa: E402
CLK = Clocks(0)

nv, ops = pkg._native, pkg.ops
dev = torch.device("cuda", 0)
PEAK = 3350.0     # GB/s: H100 SXM data sheet (HBM3)


LAST_CLOCKS = [None]


def timeit(fn, iters=10, warm=3):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for _ in range(warm):
        fn()

    def run():
        ts = []
        for _ in range(iters):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        ts.sort()
        return ts[len(ts) // 2]
    ms, LAST_CLOCKS[0] = CLK.sample_while(run)      # NVML SM clock + throttle reasons sampled during the timed loop
    return ms


def report(name, ms, npix, bpp):
    gbs = npix * bpp / ms / 1e6
    print(json.dumps({"kernel": name, "ms": round(ms, 4), "MP/s": round(npix / ms / 1e3, 1), "GB/s": round(gbs, 1), "frac_hbm": round(gbs / PEAK, 3), "clocks": LAST_CLOCKS[0]}), flush=True)


def main():
    lut = pkg.VRGDG_LUTS._parse_cube_file(os.path.join(LUTS, "B200 Vintage 33.cube"))
    lut_dev = ops.pack_lut(lut["lut"], dev)
    for (B, H, W, dt, tag) in ((16, 1080, 1920, torch.float16, "1080p_f16"), (4, 2160, 3840, torch.float32, "4k_f32"), (16, 1080, 1920, torch.float32, "1080p_f32")):
        for dist in ("nat", "white"):
            x = natural_frames(B, H, W, seed=1, dtype=dt, device=dev) if dist == "nat" else torch.rand(B, H, W, 3, device=dev).to(dt)
            npix = B * H * W
            bpp = 2 * 3 * x.element_size()
            out = torch.empty_like(x)
            report(f"copy/{tag}", timeit(lambda: out.copy_(x)), npix, bpp)
            report(f"grain/{tag}/{dist}", timeit(lambda: ops.grain(x, 0.04, 0.5, 0.5, seed=42)), npix, bpp)
            report(f"lut33/{tag}/{dist}", timeit(lambda: ops.lut3d_apply(x, lut_dev, [0, 0, 0], [1, 1, 1], 1.0, 0.0)), npix, bpp)
            report(f"unsharp_tma/{tag}/{dist}", timeit(lambda: ops.stencil3x3(x, nv.STENCIL_BOX_UNSHARP, 0.5, nv.BORDER_REPLICATE)), npix, bpp)
            os.environ["VRGDG_NO_TMA"] = "1"
            report(f"unsharp_generic/{tag}/{dist}", timeit(lambda: ops.stencil3x3(x, nv.STENCIL_BOX_UNSHARP, 0.5, nv.BORDER_REPLICATE)), npix, bpp)
            del os.environ["VRGDG_NO_TMA"]
            chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), lut=dict(lut_data=lut, strength=10.0),
                                        stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=dev)
            report(f"chain_g_l_u/{tag}/{dist}", timeit(lambda: chain(x, out=out)), npix, bpp)
            gl = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), lut=dict(lut_data=lut, strength=10.0), device=dev)
            report(f"point_g_l/{tag}/{dist}", timeit(lambda: gl(x, out=out)), npix, bpp)
            gu = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=dev)
            report(f"chain_g_u/{tag}/{dist}", timeit(lambda: gu(x, out=out)), npix, bpp)
            if dist == "nat":
                sums = None
                report(f"lab_moments/{tag}", timeit(lambda: ops.lab_moments(x)), npix, bpp / 2)
                sums = ops.lab_moments(x)
                params = ops.colormatch_params(sums, sums[:1].contiguous())
                report(f"colormatch_apply/{tag}", timeit(lambda: ops.colormatch_apply(x, params, 1.0, 0.0)), npix, bpp)
            if dist == "nat" and tag == "4k_f32":
                # configs[2] / configs[3] shapes at a reduced batch: the colour-match node path (moments + params + apply = 2 passes)
                # and the full chain grain -> colour match -> LUT -> unsharp (moments pass + fused kernel)
                ref = natural_frames(1, H, W, seed=9, dtype=dt, device=dev)
                ref_sums = ops.lab_moments(ref)
                def cm_node():
                    p = ops.colormatch_params(ops.lab_moments(x), ref_sums)
                    return ops.colormatch_apply(x, p, 1.0, 0.0)
                report(f"config3_colormatch_node/{tag}", timeit(cm_node), npix, bpp)
                full = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), colormatch=dict(ref_sums=ref_sums, strength=1.0),
                                           lut=dict(lut_data=lut, strength=10.0), stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=dev)
                report(f"config4_full_chain/{tag}", timeit(lambda: full(x, out=out)), npix, bpp)
                u8 = (x * 255).round().clamp(0, 255).to(torch.uint8)
                u8o = torch.empty_like(u8)
                report(f"chain_g_l_u/4k_u8bgr", timeit(lambda: chain(u8, out=u8o)), npix, 6)
                eff = pkg.chain.PostChain(stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5),
                                          post_grain=dict(intensity=0.04, saturation_mix=0.5, seed=42, seed_mode=nv.SEED_PER_FRAME), device=dev)
                report(f"enhancer_unsharp_grain/4k_u8bgr", timeit(lambda: eff(u8, out=u8o)), npix, 6)
                report(f"enhancer_unsharp_grain/{tag}", timeit(lambda: eff(x, out=out)), npix, bpp)
                vt = importlib.import_module("comfyui-vrgamedevgirl_b200.video_tools")
                for name, st in (("adjust_pointwise", {"temperature": 20, "exposure": 10, "contrast": 15, "saturation": 10, "highlights": -20, "fade": 10, "vignette": 30}),
                                 ("adjust_sharpen", {"contrast": 10, "sharpen": 40}), ("adjust_clarity9x9", {"contrast": 10, "clarity": 50}),
                                 ("adjust_everything", {"temperature": 20, "exposure": 10, "contrast": 15, "saturation": 10, "shadows": 20, "sharpen": 40, "clarity": 50, "fade": 10, "vignette": 30})):
                    desc = vt._adjust_desc(st, H, W)
                    report(f"{name}/{tag}", timeit(lambda: ops.adjust(x, desc)), npix, bpp)
                    report(f"{name}/4k_u8bgr", timeit(lambda: ops.adjust(u8, desc)), npix, 6)
                del u8, u8o, ref
            del x, out
            torch.cuda.empty_cache()


def resize_lines():
    """resize / restore (video_enhance): GPx/s counts OUTPUT pixels; bytes = source + output frames."""
    for dt, tag in ((torch.float32, "f32"), (torch.float16, "f16")):
        small = natural_frames(8, 1080, 1920, seed=3, dtype=dt, device=dev)
        big = natural_frames(2, 2160, 3840, seed=4, dtype=dt, device=dev)
        es = small.element_size()
        for mode in ("nearest", "bilinear", "bicubic", "area"):
            nout = 8 * 2160 * 3840
            ms = timeit(lambda: ops.resize(small, 2160, 3840, mode), iters=6, warm=2)
            report(f"resize_{mode}_up2x/8x1080p_{tag}", ms, nout, 3 * es * 1.25)
            nout = 2 * 1080 * 1920
            ms = timeit(lambda: ops.resize(big, 1080, 1920, mode), iters=6, warm=2)
            report(f"resize_{mode}_down2x/2x4k_{tag}", ms, nout, 3 * es * 5)
        a = natural_frames(4, 2160, 3840, seed=5, dtype=dt, device=dev)
        b = natural_frames(4, 2160, 3840, seed=6, dtype=dt, device=dev)
        report(f"restore_blend/4x4k_{tag}", timeit(lambda: ops.blend(a, b, 0.35, 0.65)), 4 * 2160 * 3840, 9 * es)
        del small, big, a, b
        torch.cuda.empty_cache()
    u = (natural_frames(8, 1080, 1920, seed=7, device=dev) * 255).to(torch.uint8)
    report("lanczos4_u8_up2x/8x1080p", timeit(lambda: ops.resize_lanczos4_u8(u, 2160, 3840), iters=6, warm=2), 8 * 2160 * 3840, 3 * 1.25)
    report("lanczos4_u8_up1.5x/8x720p", timeit(lambda: ops.resize_lanczos4_u8(u[:, :720, :1280].contiguous(), 1080, 1920), iters=6, warm=2), 8 * 1080 * 1920, 3 * (1 + 1 / 2.25))
    u4 = (natural_frames(2, 2160, 3840, seed=8, device=dev) * 255).to(torch.uint8)
    report("lanczos4_u8_down2x/2x4k", timeit(lambda: ops.resize_lanczos4_u8(u4, 1080, 1920), iters=6, warm=2), 2 * 1080 * 1920, 3 * 5)


if __name__ == "__main__":
    if "--resize-only" not in sys.argv:
        main()
    resize_lines()

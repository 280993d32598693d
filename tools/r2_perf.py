"""Round-2 scratch micro-benchmark (GPU box only; NOT the contract bench): the kernels of the headline chain and the LUT sizes the
reference ships, every line with an NVML clock record.   python tools/r2_perf.py [rows...]
rows: cm (colour-match kernels + full chain), chains (fused chains without colour match), luts (33/64/65 natural + white)"""
import importlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
pkg = importlib.import_module("comfyui-vrgamedevgirl_b200")
from helpers import LUTS, natural_frames, write_big_cube  # noqa: E402
from _clocks import Clocks  # noqa: E402

nv, ops = pkg._native, pkg.ops
dev = torch.device("cuda", 0)
PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0   # H100 SXM data sheet
CLK = Clocks(0)


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
    return CLK.sample_while(run)


def report(name, res, npix, bpp):
    ms, clocks = res
    gbs = npix * bpp / ms / 1e6
    print(json.dumps({"kernel": name, "ms": round(ms, 4), "MP/s": round(npix / ms / 1e3, 1), "GB/s": round(gbs, 1), "frac_hbm": round(gbs / PEAK, 3),
                      "clocks": clocks}), flush=True)


def lut33():
    return pkg.VRGDG_LUTS._parse_cube_file(os.path.join(LUTS, "B200 Vintage 33.cube"))


def rows_cm():
    lut = lut33()
    for (B, H, W, dt, tag) in ((32, 2160, 3840, torch.float32, "4k_f32"), (64, 1080, 1920, torch.float32, "1080p_f32"), (8, 2160, 3840, torch.float16, "4k_f16")):
        x = natural_frames(8, H, W, seed=1, dtype=dt, device=dev).repeat(B // 8, 1, 1, 1).contiguous()
        out = torch.empty_like(x)
        npix, bpp = B * H * W, 2 * 3 * x.element_size()
        ref_sums = ops.lab_moments(natural_frames(1, H, W, seed=9, dtype=dt, device=dev))
        report(f"lab_moments/{tag}", timeit(lambda: ops.lab_moments(x)), npix, bpp / 2)
        d = nv.ChainDesc()
        d.grain_enabled, d.grain_intensity, d.grain_sat, d.grain_one_minus_sat, d.grain_seed = 1, 0.04, 0.5, 0.5, 42
        report(f"lab_moments_of_grain/{tag}", timeit(lambda: ops.chain_lab_moments(x, d)), npix, bpp / 2)
        params = ops.colormatch_params(ops.lab_moments(x), ref_sums)
        report(f"colormatch_apply/{tag}", timeit(lambda: ops.colormatch_apply(x, params, 1.0, 0.0)), npix, bpp)
        node = pkg.ColorMatchToReference()
        report(f"colormatch_node_path/{tag}", timeit(lambda: ops.colormatch_apply(x, ops.colormatch_params(ops.lab_moments(x), ref_sums), 1.0, 0.0)), npix, bpp)
        full = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), colormatch=dict(ref_sums=ref_sums, strength=1.0),
                                   lut=dict(lut_data=lut, strength=10.0), stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=dev)
        report(f"full_chain_g_cm_l_u/{tag}", timeit(lambda: full(x, out=out)), npix, bpp)
        for g in (1, 2, 4, 8):
            if g > B:
                continue
            full.group_frames = g
            report(f"full_chain_g_cm_l_u/{tag}/planes_G{g}", timeit(lambda: full(x, out=out)), npix, bpp)
            full.recompute = True
            report(f"full_chain_g_cm_l_u/{tag}/recompute_G{g}", timeit(lambda: full(x, out=out)), npix, bpp)
            full.recompute = False
        full.group_frames, full.serial = 0, True
        report(f"full_chain_g_cm_l_u/{tag}/serial", timeit(lambda: full(x, out=out)), npix, bpp)
        full.serial = False
        full.group_frames, full.split = 0, True
        report(f"full_chain_g_cm_l_u/{tag}/three_calls", timeit(lambda: full(x, out=out)), npix, bpp)
        full.split = False
        cmonly = pkg.chain.PostChain(colormatch=dict(ref_sums=ref_sums, strength=1.0), device=dev)
        for g in (0, 1, 2, 4):
            cmonly.group_frames = g
            report(f"colormatch_one_call/{tag}/planes_G{g}", timeit(lambda: cmonly(x, out=out)), npix, bpp)
        cmonly.recompute, cmonly.group_frames = True, 1
        report(f"colormatch_one_call/{tag}/recompute_G1", timeit(lambda: cmonly(x, out=out)), npix, bpp)
        cmu = pkg.chain.PostChain(colormatch=dict(ref_sums=ref_sums, strength=1.0), stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=dev)
        report(f"chain_cm_u/{tag}", timeit(lambda: cmu(x, out=out)), npix, bpp)
        del x, out, node
        torch.cuda.empty_cache()


def rows_ext():
    """the two labelled extensions: histogram / CDF colour match and the temporal 3-frame sharpen"""
    for (B, H, W, dt, tag) in ((8, 2160, 3840, torch.float32, "4k_f32"), (32, 1080, 1920, torch.float32, "1080p_f32")):
        x = natural_frames(8, H, W, seed=1, dtype=dt, device=dev).repeat(B // 8, 1, 1, 1).contiguous()
        npix, bpp = B * H * W, 2 * 3 * x.element_size()
        ref_counts = ops.hist_counts(natural_frames(1, H, W, seed=9, dtype=dt, device=dev))
        report(f"hist_counts/{tag}", timeit(lambda: ops.hist_counts(x)), npix, bpp / 2)
        counts = ops.hist_counts(x)
        tables = ops.histmatch_tables(counts, ref_counts)
        report(f"histmatch_apply/{tag}", timeit(lambda: ops.histmatch_apply(x, tables, 1.0, 0.0)), npix, bpp)
        report(f"histmatch_whole/{tag}", timeit(lambda: ops.histmatch_apply(x, ops.histmatch_tables(ops.hist_counts(x), ref_counts), 1.0, 0.0)), npix, bpp)
        report(f"temporal_sharpen/{tag}", timeit(lambda: ops.temporal_sharpen(x, 0.5)), npix, bpp)
        del x
        torch.cuda.empty_cache()


def rows_chains():
    lut = lut33()
    for (B, H, W, dt, tag) in ((4, 2160, 3840, torch.float32, "4k_f32"), (16, 1080, 1920, torch.float16, "1080p_f16")):
        for dist in ("nat", "white"):
            x = natural_frames(B, H, W, seed=1, dtype=dt, device=dev) if dist == "nat" else torch.rand(B, H, W, 3, device=dev).to(dt)
            out = torch.empty_like(x)
            npix, bpp = B * H * W, 2 * 3 * x.element_size()
            report(f"copy/{tag}", timeit(lambda: out.copy_(x)), npix, bpp)
            report(f"grain/{tag}/{dist}", timeit(lambda: ops.grain(x, 0.04, 0.5, 0.5, seed=42)), npix, bpp)
            report(f"unsharp/{tag}/{dist}", timeit(lambda: ops.stencil3x3(x, nv.STENCIL_BOX_UNSHARP, 0.5, nv.BORDER_REPLICATE)), npix, bpp)
            chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), lut=dict(lut_data=lut, strength=10.0),
                                        stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=dev)
            report(f"chain_g_l_u/{tag}/{dist}", timeit(lambda: chain(x, out=out)), npix, bpp)
            gu = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=dev)
            report(f"chain_g_u/{tag}/{dist}", timeit(lambda: gu(x, out=out)), npix, bpp)
            del x, out
            torch.cuda.empty_cache()


def rows_luts():
    import tempfile
    tables = {33: lut33()}
    with tempfile.TemporaryDirectory() as tmp:
        for s in (64, 65):
            tables[s] = pkg.VRGDG_LUTS._parse_cube_file(write_big_cube(os.path.join(tmp, "big_%d.cube" % s), s))
    for (B, H, W, dt, tag) in ((4, 2160, 3840, torch.float32, "4k_f32"), (16, 1080, 1920, torch.float16, "1080p_f16")):
        for dist in ("nat", "white"):
            x = natural_frames(B, H, W, seed=1, dtype=dt, device=dev) if dist == "nat" else torch.rand(B, H, W, 3, device=dev).to(dt)
            out = torch.empty_like(x)
            npix, bpp = B * H * W, 2 * 3 * x.element_size()
            for s, data in tables.items():
                packed = ops.pack_lut(data["lut"], dev)
                report(f"lut{s}/{tag}/{dist}", timeit(lambda: ops.lut3d_apply(x, packed, [0, 0, 0], [1, 1, 1], 1.0, 0.0)), npix, bpp)
                chain = pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42), lut=dict(lut_data=data, strength=10.0),
                                            stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), device=dev)
                report(f"chain_g_l{s}_u/{tag}/{dist}", timeit(lambda: chain(x, out=out)), npix, bpp)
            del x, out
            torch.cuda.empty_cache()


if __name__ == "__main__":
    want = sys.argv[1:] or ["cm", "chains", "luts"]
    if "cm" in want:
        rows_cm()
    if "chains" in want:
        rows_chains()
    if "luts" in want:
        rows_luts()
    if "ext" in want:
        rows_ext()

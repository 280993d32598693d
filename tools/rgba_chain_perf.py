"""3D LUT -> 3x3 unsharp on RGBA frames: the one-pass chain (vrgdg_chain_apply_ch) vs the two-kernel composition
(vrgdg_lut3d_apply with 4 channels, then vrgdg_stencil3x3_ch) vs the RGB fused chain at the same pixel count, on device-resident
frames of the sizes a user runs; then one host -> host line, VRGDG_B200_PostChain vs VRGDG_LUTS -> FastUnsharpSharpen.

    python tools/rgba_chain_perf.py [--rounds 8] [--iters 10] [--warmup 3] [--host-rounds 3] [--out FILE]

Device workloads: 16 x 3840x2160 fp32 and 64 x 1920x1080 fp16, LUT "B200 Vintage 33.cube" at strength 10, unsharp 0.5 with the
NumPy-path (edge-replicated) border.  Within every round the three configurations alternate (order rotated every round), each
timed with CUDA events over --iters back-to-back calls, so clock and neighbour noise hit them alike.  Per workload and
configuration: median / min / max ms per call over the rounds, GPx/s, and the algorithmic bytes (one read and one write of the
frames: RGBA 32 / 16 B/px, RGB 24 / 12 B/px for fp32 / fp16; the composition moves twice the RGBA figure) over the median time as a
fraction of the H100 SXM data sheet's 3.35 TB/s.  Before timing, the fused result is compared with the composition (fp32: bit for
bit; fp16: max |diff|, the composition rounds the LUT result to 16 bits in between) and its RGB channels with the RGB chain.
Host line: 16 x 1920x1080 fp32 pageable RGBA frames, node vs the two stock nodes, alternating, host clock around each call (each
ends with its result on the host).  The card's name, power limit and the SM clock record of the timed region are printed in the
same run."""
import argparse
import ctypes
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _clocks import Clocks  # noqa: E402

PKG = "comfyui-vrgamedevgirl_b200"
PEAK = 3.35e12
LUT = "B200 Vintage 33.cube"
WORKLOADS = {"16x4K_fp32": (16, 2160, 3840, torch.float32), "64x1080p_fp16": (64, 1080, 1920, torch.float16)}
HOST = (16, 1080, 1920)
CONFIGS = ("fused_rgba", "composition_rgba", "fused_rgb")


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        txt = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=60).stdout
    except (OSError, subprocess.SubprocessError) as e:
        return {"nvidia-smi": "unavailable: %s" % e}
    return dict(zip(q.split(","), (f.strip() for f in txt.strip().split(","))))


def emit(lines, line):
    lines.append(line)
    print(json.dumps(line), flush=True)


def device_workload(pkg, lib, dev, name, B, H, W, dt, args, clocks, lines):
    nv = pkg._native
    stream = nv.stream_ptr(dev)
    g = torch.Generator(device=dev).manual_seed(7)
    x4 = torch.rand(B, H, W, 4, device=dev, generator=g).to(dt)
    x3 = x4[..., :3].contiguous()
    o4, tmp, oc, o3 = torch.empty_like(x4), torch.empty_like(x4), torch.empty_like(x4), torch.empty_like(x3)
    chain = pkg.chain.PostChain(lut=dict(lut_data=pkg.VRGDG_LUTS._load_lut(LUT), strength=10.0),
                                stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5, border=nv.BORDER_REPLICATE), device=dev)
    d = chain._desc(x4, 0, [])
    code = nv.DTYPE_CODE[dt]

    def call(cfg):
        if cfg == "fused_rgba":
            nv.check(lib.vrgdg_chain_apply_ch(nv.ptr(x4), nv.ptr(o4), B, H, W, 4, code, ctypes.byref(d), stream))
        elif cfg == "composition_rgba":
            nv.check(lib.vrgdg_lut3d_apply(nv.ptr(x4), nv.ptr(tmp), B * H * W, 4, code, d.lut, d.lut_size, d.lut_dmin, d.lut_dspan,
                                           ctypes.c_float(d.lut_blend), ctypes.c_float(d.lut_one_minus_blend), stream))
            nv.check(lib.vrgdg_stencil3x3_ch(nv.ptr(tmp), nv.ptr(oc), B, H, W, 4, code, d.stencil_op, ctypes.c_float(d.stencil_strength),
                                             d.stencil_border, stream))
        else:
            nv.check(lib.vrgdg_chain_apply(nv.ptr(x3), nv.ptr(o3), B, H, W, code, ctypes.byref(d), stream))
    for cfg in CONFIGS:
        for _ in range(args.warmup):
            call(cfg)
    torch.cuda.synchronize()
    checks = {"fused_equals_composition": torch.equal(o4, oc),
              "fused_vs_composition_max_abs_diff": float((o4.float() - oc.float()).abs().max()),
              "rgb_channels_equal_rgb_chain": torch.equal(o4[..., :3], o3)}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed():
        ms = {c: [] for c in CONFIGS}
        for r in range(args.rounds):
            k = r % len(CONFIGS)
            for cfg in CONFIGS[k:] + CONFIGS[:k]:
                ev0.record()
                for _ in range(args.iters):
                    call(cfg)
                ev1.record()
                ev1.synchronize()
                ms[cfg].append(ev0.elapsed_time(ev1) / args.iters)
        return ms
    ms, clk = clocks.sample_while(timed)
    px = B * H * W
    es = torch.tensor([], dtype=dt).element_size()
    for cfg in CONFIGS:
        med = statistics.median(ms[cfg])
        bpp = 2 * (3 if cfg == "fused_rgb" else 4) * es
        emit(lines, {"workload": name, "config": cfg, "frames": [B, H, W, 3 if cfg == "fused_rgb" else 4], "ms_median": round(med, 4),
                     "ms_min": round(min(ms[cfg]), 4), "ms_max": round(max(ms[cfg]), 4), "gpx_per_s": round(px / med / 1e6, 2),
                     "algorithmic_bytes_per_px": bpp, "fraction_of_3.35TBps": round(px * bpp / (med * 1e-3) / PEAK, 3),
                     **checks, "sm_clock": clk})


def host_line(pkg, args, lines):
    B, H, W = HOST
    g = torch.Generator().manual_seed(11)
    x = torch.rand(B, H, W, 4, generator=g)                  # pageable
    node = pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_PostChain"]()
    lut_node, sharpen = pkg.VRGDG_LUTS(), pkg.FastUnsharpSharpen()
    runs = {"node": lambda: node.apply_chain(x, 0.0, 0.5, 1.0, LUT, 10.0, "unsharp", 0.5, False, 8)[0],
            "stock_nodes": lambda: sharpen.apply_unsharp(lut_node.apply_lut(x, LUT, "auto", 10.0)[0], 0.5, False)[0]}
    outs = {k: f() for k, f in runs.items()}               # warm-up
    torch.cuda.synchronize()
    same = torch.equal(outs["node"], outs["stock_nodes"])
    s = {k: [] for k in runs}
    for r in range(args.host_rounds):
        for k in (("node", "stock_nodes") if r % 2 == 0 else ("stock_nodes", "node")):
            t0 = time.perf_counter()
            out = runs[k]()
            torch.cuda.synchronize()
            s[k].append(time.perf_counter() - t0)
            assert out.device.type == "cpu"
    emit(lines, {"workload": "host_%dx%dx%d_fp32_rgba_pageable" % HOST, "node_s_median": round(statistics.median(s["node"]), 4),
                 "stock_nodes_s_median": round(statistics.median(s["stock_nodes"]), 4), "node_s": [round(v, 4) for v in s["node"]],
                 "stock_nodes_s": [round(v, 4) for v in s["stock_nodes"]], "node_equals_stock_nodes": same})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--iters", type=int, default=10, help="calls per timing")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has nothing to report without one")
    pkg = importlib.import_module(PKG)
    lib = pkg._native.load_library()
    dev = torch.device("cuda", 0)
    lines = []
    emit(lines, {"card": card(), "device": torch.cuda.get_device_name(dev), "torch": torch.__version__, "cuda": torch.version.cuda})
    clocks = Clocks(0)
    for name, (B, H, W, dt) in WORKLOADS.items():
        device_workload(pkg, lib, dev, name, B, H, W, dt, args, clocks, lines)
        torch.cuda.empty_cache()
    host_line(pkg, args, lines)
    if args.out:
        with open(args.out, "w", encoding="utf-8") as fh:
            fh.write("\n".join(json.dumps(l) for l in lines) + "\n")


if __name__ == "__main__":
    main()

"""RGB vs RGBA 3x3 unsharp (vrgdg_stencil3x3_ch, NumPy-path border) on device-resident frames of the sizes a user runs.

    python tools/rgba_stencil_perf.py [--rounds 8] [--iters 10] [--warmup 3] [--out FILE]

Workloads: 16 x 3840x2160 fp32 and 64 x 1920x1080 fp16.  Within every round the two layouts alternate (order flipped every other
round), each timed with CUDA events over --iters back-to-back calls, so clock and neighbour noise hit both alike.  Per workload and
layout: median / min / max ms per call over the rounds, GPx/s, and the algorithmic bytes (one read and one write of the frames:
RGB 24 / 12 B/px, RGBA 32 / 16 B/px for fp32 / fp16) over the median time as a fraction of the H100 SXM data sheet's 3.35 TB/s.
Before timing, the RGBA result's RGB channels are checked bit for bit against the RGB kernel on the same pixels.  The card's name,
power limit and the SM clock record of the timed region are printed in the same run."""
import argparse
import ctypes
import importlib
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _clocks import Clocks  # noqa: E402

PKG = "comfyui-vrgamedevgirl_b200"
PEAK = 3.35e12
WORKLOADS = {"16x4K_fp32": (16, 2160, 3840, torch.float32), "64x1080p_fp16": (64, 1080, 1920, torch.float16)}


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        txt = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=60).stdout
    except (OSError, subprocess.SubprocessError) as e:
        return {"nvidia-smi": "unavailable: %s" % e}
    return dict(zip(q.split(","), (f.strip() for f in txt.strip().split(","))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--iters", type=int, default=10, help="calls per timing")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has nothing to report without one")
    pkg = importlib.import_module(PKG)
    nv = pkg._native
    lib = nv.load_library()
    dev = torch.device("cuda", 0)
    lines = [{"card": card(), "device": torch.cuda.get_device_name(dev), "torch": torch.__version__, "cuda": torch.version.cuda}]
    print(json.dumps(lines[0]), flush=True)
    clocks = Clocks(0)
    stream = nv.stream_ptr(dev)

    for name, (B, H, W, dt) in WORKLOADS.items():
        g = torch.Generator(device=dev).manual_seed(7)
        x4 = torch.rand(B, H, W, 4, device=dev, generator=g).to(dt)
        x3 = x4[..., :3].contiguous()
        frames = {3: (x3, torch.empty_like(x3)), 4: (x4, torch.empty_like(x4))}

        def call(c):
            src, dst = frames[c]
            nv.check(lib.vrgdg_stencil3x3_ch(nv.ptr(src), nv.ptr(dst), B, H, W, c, nv.DTYPE_CODE[dt], nv.STENCIL_BOX_UNSHARP,
                                             ctypes.c_float(0.5), nv.BORDER_REPLICATE, stream))
        for c in (3, 4):
            for _ in range(args.warmup):
                call(c)
        torch.cuda.synchronize()
        same = torch.equal(frames[4][1][..., :3], frames[3][1])
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def timed():
            ms = {3: [], 4: []}
            for r in range(args.rounds):
                for c in ((3, 4) if r % 2 == 0 else (4, 3)):
                    ev0.record()
                    for _ in range(args.iters):
                        call(c)
                    ev1.record()
                    ev1.synchronize()
                    ms[c].append(ev0.elapsed_time(ev1) / args.iters)
            return ms
        ms, clk = clocks.sample_while(timed)
        px = B * H * W
        for c in (3, 4):
            med = statistics.median(ms[c])
            bpp = 2 * c * torch.tensor([], dtype=dt).element_size()
            line = {"workload": name, "layout": "RGB" if c == 3 else "RGBA", "frames": [B, H, W, c], "ms_median": round(med, 4),
                    "ms_min": round(min(ms[c]), 4), "ms_max": round(max(ms[c]), 4), "gpx_per_s": round(px / med / 1e6, 2),
                    "algorithmic_bytes_per_px": bpp, "fraction_of_3.35TBps": round(px * bpp / (med * 1e-3) / PEAK, 3),
                    "rgb_channels_equal_rgb_kernel": same, "sm_clock": clk}
            lines.append(line)
            print(json.dumps(line), flush=True)
        del frames, x3, x4
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w", encoding="utf-8") as fh:
            fh.write("\n".join(json.dumps(l) for l in lines) + "\n")


if __name__ == "__main__":
    main()

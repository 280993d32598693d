"""The Video Enhance restore: the fused vrgdg_restore_blend pass against the resize -> blend composition it replaced.

    python tools/restore_perf.py [--rounds 8] [--iters 5] [--warmup 2] [--host-frames 64] [--host-rounds 3] [--out FILE]

1. Device-resident: 16 x 3840x2160 fp32 originals restored from 16 enhanced frames, bicubic, strength 0.7, in two geometries:
   "stretch" (1920x1080 enhanced frames) and "letterbox_roi" (1920x1088 working frames whose 1920x1080 content is the ROI).  The
   composition (ops.resize -> ops.blend into originals.clamp(0, 1)) and the fused launch alternate within every round (order
   flipped every other round), each timed with CUDA events over --iters calls.  Per variant: median / min / max ms, GPx/s, and the
   algorithmic bytes (originals read once, output written once, enhanced frames read once) over the median time as a fraction of
   the H100 SXM data sheet's 3.35 TB/s.  The two results are compared with torch.equal first.
2. Host -> host through the node's restore_frames: --host-frames pageable 4K fp32 originals (1080p enhanced) with the whole-clip
   path the package used before (upload everything, compose, download) and the streamed one, on one device and with
   VRGDG_DEVICES=all, alternating; wall time around each call (each ends with the result on the host).
3. Peak device memory (torch.cuda.max_memory_allocated growth) of the old and new host -> host paths on the same clip.
The card's name, power limit and the SM clock record of the timed region are printed in the same run."""
import argparse
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
B, H, W = 16, 2160, 3840
GEOMETRIES = {"stretch": ("Stretch to dimensions", 1080, 1920), "letterbox_roi": ("Fit with letterbox (preserve all)", 1088, 1920)}
STRENGTH = 0.7


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        txt = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=60).stdout
    except (OSError, subprocess.SubprocessError) as e:
        return {"nvidia-smi": "unavailable: %s" % e}
    return dict(zip(q.split(","), (f.strip() for f in txt.strip().split(","))))


def composition(ops, enh, orig, roi, s):
    """the arithmetic restore_frames ran before the fused kernel: a full-size resample, a clamped copy, a blend temporary"""
    restored = ops.resize(enh, int(orig.shape[1]), int(orig.shape[2]), "bicubic", roi=roi).to(orig.dtype)
    out = orig.clamp(0, 1)
    out[..., :3] = ops.blend(orig[..., :3], restored, 1.0 - s, s)
    return out


def old_restore_frames(ve, ops, rt, originals, enhanced, fit, s):
    """restore_frames as the package ran it before streaming: the whole clip on one device"""
    dev = rt.compute_device(originals)
    orig = rt.upload(originals, dev)
    restored = ve._restore_batch(rt.upload(enhanced, dev), int(orig.shape[2]), int(orig.shape[1]), fit, "Bicubic (recommended)").to(orig.dtype)
    n = min(int(orig.shape[0]), int(restored.shape[0]))
    out = orig.clamp(0, 1)
    out[:n, ..., :3] = ops.blend(orig[:n, ..., :3], restored[:n], 1.0 - s, s)
    return out.to(originals.device)


def emit(lines, line):
    lines.append(line)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--iters", type=int, default=5, help="calls per timing")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-frames", type=int, default=64)
    ap.add_argument("--host-rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has nothing to report without one")
    pkg = importlib.import_module(PKG)
    ops = pkg.ops
    ve = importlib.import_module(PKG + ".video_enhance")
    rt = importlib.import_module(PKG + "._runtime")
    dev = torch.device("cuda", 0)
    lines = []
    emit(lines, {"card": card(), "device": torch.cuda.get_device_name(dev), "visible_devices": torch.cuda.device_count(),
                 "torch": torch.__version__, "cuda": torch.version.cuda})
    clocks = Clocks(0)

    # ---- 1. device-resident ----
    g = torch.Generator(device=dev).manual_seed(7)
    orig = torch.rand(B, H, W, 3, device=dev, generator=g) * 1.2 - 0.1
    for name, (fit, He, We) in GEOMETRIES.items():
        enh = torch.rand(B, He, We, 3, device=dev, generator=g)
        roi = ve._restore_roi(We, He, W, H, fit)
        calls = {"composition": lambda: composition(ops, enh, orig, roi, STRENGTH),
                 "fused": lambda: ops.restore_blend(enh, orig, "bicubic", 1.0 - STRENGTH, STRENGTH, roi=roi)}
        for f in calls.values():
            for _ in range(args.warmup):
                f()
        torch.cuda.synchronize()
        equal = torch.equal(calls["fused"](), calls["composition"]())
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def timed():
            ms = {k: [] for k in calls}
            for r in range(args.rounds):
                for k in (("composition", "fused") if r % 2 == 0 else ("fused", "composition")):
                    ev0.record()
                    for _ in range(args.iters):
                        calls[k]()
                    ev1.record()
                    ev1.synchronize()
                    ms[k].append(ev0.elapsed_time(ev1) / args.iters)
            return ms
        ms, clk = clocks.sample_while(timed)
        px = B * H * W
        nbytes = 2 * px * 3 * 4 + B * roi[2] * roi[3] * 3 * 4     # originals + output + the enhanced ROI, each once
        for k in calls:
            med = statistics.median(ms[k])
            emit(lines, {"workload": "device_16x4K_fp32_" + name, "variant": k, "enhanced": [B, He, We, 3], "roi": list(roi),
                         "ms_median": round(med, 3), "ms_min": round(min(ms[k]), 3), "ms_max": round(max(ms[k]), 3),
                         "gpx_per_s": round(px / med / 1e6, 2), "algorithmic_bytes": nbytes,
                         "fraction_of_3.35TBps": round(nbytes / (med * 1e-3) / PEAK, 3), "fused_equals_composition": equal,
                         "sm_clock": clk})
        del enh, calls
    del orig
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

    # ---- 2 / 3. host -> host ----
    n = args.host_frames
    cpu = torch.Generator().manual_seed(9)
    originals = torch.rand(n, H, W, 3, generator=cpu)
    enhanced = torch.rand(n, 1080, 1920, 3, generator=cpu)
    fit = "Stretch to dimensions"
    cards = [torch.device("cuda", i) for i in range(torch.cuda.device_count()) if tuple(torch.cuda.get_device_capability(i)) == (9, 0)]
    variants = {
        "old_whole_clip": lambda: old_restore_frames(ve, ops, rt, originals, enhanced, fit, STRENGTH),
        "streamed_one_device": lambda: ve.restore_frames(originals, enhanced, W, H, fit, "Bicubic (recommended)", STRENGTH),
        "streamed_vrgdg_devices_all": lambda: ve.restore_frames(originals, enhanced, W, H, fit, "Bicubic (recommended)", STRENGTH),
    }

    def run(k):
        if k == "streamed_vrgdg_devices_all":
            os.environ["VRGDG_DEVICES"] = "all"
        else:
            os.environ.pop("VRGDG_DEVICES", None)
        for c in cards:
            torch.cuda.synchronize(c)
            torch.cuda.reset_peak_memory_stats(c)
        base = [torch.cuda.memory_allocated(c) for c in cards]
        t0 = time.perf_counter()
        out = variants[k]()
        for c in cards:
            torch.cuda.synchronize(c)
        dt = time.perf_counter() - t0
        peak = max(torch.cuda.max_memory_allocated(c) - b for c, b in zip(cards, base))
        return out, dt, peak
    ref = None
    results = {k: {"s": [], "peak": 0, "equal": True} for k in variants}
    for r in range(args.host_rounds + 1):                     # round 0 warms every path up and is not reported
        for k in (list(variants) if r % 2 == 0 else list(reversed(list(variants)))):
            out, dt, peak = run(k)
            if ref is None:
                ref = out
            elif r == 0:
                results[k]["equal"] = bool(torch.equal(out, ref))
            if r > 0:
                results[k]["s"].append(dt)
                results[k]["peak"] = max(results[k]["peak"], peak)
            del out
    os.environ.pop("VRGDG_DEVICES", None)
    clip = originals.numel() * originals.element_size()
    for k, v in results.items():
        med = statistics.median(v["s"])
        emit(lines, {"workload": "host_%dx4K_fp32_pageable" % n, "variant": k, "devices": len(cards) if k.endswith("all") else 1,
                     "s_median": round(med, 3), "s_min": round(min(v["s"]), 3), "s_max": round(max(v["s"]), 3),
                     "frames_per_s": round(n / med, 1), "peak_device_bytes": v["peak"], "peak_over_clip": round(v["peak"] / clip, 3),
                     "equals_old_path": v["equal"]})
    if args.out:
        with open(args.out, "w", encoding="utf-8") as fh:
            fh.write("\n".join(json.dumps(l) for l in lines) + "\n")


if __name__ == "__main__":
    main()

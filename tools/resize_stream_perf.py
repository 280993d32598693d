"""The Video Enhance resample helpers host -> host: the whole-clip _resize_batch the package ran before against the streamed one.

    python tools/resize_stream_perf.py [--frames 64] [--rounds 3] [--out FILE]

Two workloads of pageable fp32 host frames, bicubic, "Crop to fill" (same aspect ratio, so no crop happens):
  * prepare: --frames x 3840x2160 -> 1280x720;
  * upscale: --frames x 1920x1080 -> 3840x2160 (the README's example).
Three variants per workload, alternating within every round (order reversed every other round), after one warm-up round:
  * old_whole_clip: upload the whole clip (through a pinned staging copy of it), one launch, download into a pageable tensor;
  * streamed_one_device: _resize_batch with VRGDG_DEVICES unset;
  * streamed_vrgdg_devices_all: _resize_batch with VRGDG_DEVICES=all, whatever cards are visible.
Per variant: wall time around the call (each ends with the result on the host), the growth of torch.cuda.max_memory_allocated over
the call (the largest over the cards), the peak of pinned host bytes handed out during the call (torch.cuda.host_memory_stats,
"active_bytes"; torch's pinned allocator rounds each block up to a power of two, and the count includes a pinned result), whether
the result is pinned, and torch.equal against the old path's result.  The card's name and power limit are read in the same run."""
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

PKG = "comfyui-vrgamedevgirl_b200"
WORKLOADS = {"prepare_4K_to_720p": ((2160, 3840), (1280, 720)), "upscale_1080p_to_4K": ((1080, 1920), (3840, 2160))}
FIT, METHOD = "Crop to fill", "Bicubic (recommended)"


def cards_info():
    q = "index,name,power.limit,clocks.max.sm"
    try:
        txt = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
    except (OSError, subprocess.SubprocessError) as e:
        return [{"nvidia-smi": "unavailable: %s" % e}]
    return [dict(zip(q.split(","), (f.strip() for f in line.split(",")))) for line in txt.strip().splitlines()]


def old_resize_batch(ve, ops, rt, images, tw, th, fit, method):
    """_resize_batch as the package ran it before streaming: the whole clip uploaded, one launch, one download"""
    dev = rt.compute_device(images)
    src = rt.upload(images, dev)
    x0, y0, sw, sh = 0, 0, int(src.shape[2]), int(src.shape[1])
    resampled, offset = ve._resize_plan(sw, sh, tw, th, fit)
    ow, oh = ve._output_size(resampled, offset, tw, th, fit)
    out = ops.resize(src, oh, ow, ve._interpolation(method), roi=(x0, y0, sw, sh), resampled=resampled, offset=offset)
    return out.to(images.device)


def pinned_active():
    if not hasattr(torch.cuda, "host_memory_stats"):
        return None
    return int(torch.cuda.host_memory_stats().get("active_bytes.current", 0))


def emit(lines, line):
    lines.append(line)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has nothing to report without one")
    pkg = importlib.import_module(PKG)
    ve = importlib.import_module(PKG + ".video_enhance")
    rt = importlib.import_module(PKG + "._runtime")
    os.environ.pop("VRGDG_DEVICES", None)
    os.environ.pop("VRGDG_STREAM_CHUNK_BYTES", None)
    cards = [torch.device("cuda", i) for i in range(torch.cuda.device_count()) if tuple(torch.cuda.get_device_capability(i)) == (9, 0)]
    lines = []
    emit(lines, {"cards": cards_info(), "device": torch.cuda.get_device_name(0), "visible_devices": torch.cuda.device_count(),
                 "torch": torch.__version__, "cuda": torch.version.cuda,
                 "pinned_host_stats": "torch.cuda.host_memory_stats" if hasattr(torch.cuda, "host_memory_stats") else "not measured"})

    for wname, ((H, W), (tw, th)) in WORKLOADS.items():
        n = args.frames
        images = torch.rand(n, H, W, 3, generator=torch.Generator().manual_seed(H))
        variants = {
            "old_whole_clip": lambda: old_resize_batch(ve, pkg.ops, rt, images, tw, th, FIT, METHOD),
            "streamed_one_device": lambda: ve._resize_batch(images, tw, th, FIT, METHOD),
            "streamed_vrgdg_devices_all": lambda: ve._resize_batch(images, tw, th, FIT, METHOD),
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
            pin0 = pinned_active()
            if pin0 is not None:
                torch.cuda.reset_peak_host_memory_stats()
            t0 = time.perf_counter()
            out = variants[k]()
            for c in cards:
                torch.cuda.synchronize(c)
            dt = time.perf_counter() - t0
            peak = max(torch.cuda.max_memory_allocated(c) - b for c, b in zip(cards, base))
            pin = None if pin0 is None else int(torch.cuda.host_memory_stats()["active_bytes.peak"]) - pin0
            return out, dt, peak, pin

        ref = None
        results = {k: {"s": [], "peak": 0, "pinned": 0, "equal": True, "result_pinned": None} for k in variants}
        for r in range(args.rounds + 1):                       # round 0 warms every path up and is not timed
            for k in (list(variants) if r % 2 == 0 else list(reversed(list(variants)))):
                out, dt, peak, pin = run(k)
                if ref is None:
                    ref = out                                  # round 0 runs old_whole_clip first
                else:
                    results[k]["equal"] = results[k]["equal"] and bool(torch.equal(out, ref))
                results[k]["result_pinned"] = bool(out.is_pinned())
                if r > 0:
                    results[k]["s"].append(dt)
                    results[k]["peak"] = max(results[k]["peak"], peak)
                    results[k]["pinned"] = None if pin is None else max(results[k]["pinned"], pin)
                del out
        os.environ.pop("VRGDG_DEVICES", None)
        clip_in = images.numel() * images.element_size()
        clip_out = ref.numel() * ref.element_size()
        for k, v in results.items():
            med = statistics.median(v["s"])
            emit(lines, {"workload": "host_%d_%s_fp32_pageable" % (n, wname), "variant": k, "source": [n, H, W, 3], "target": [th, tw],
                         "devices": len(cards) if k.endswith("all") else 1,
                         "s_median": round(med, 3), "s_min": round(min(v["s"]), 3), "s_max": round(max(v["s"]), 3),
                         "frames_per_s": round(n / med, 1), "peak_device_bytes": v["peak"],
                         "peak_device_over_input_plus_output": round(v["peak"] / (clip_in + clip_out), 3),
                         "peak_pinned_host_bytes": "not measured" if v["pinned"] is None else v["pinned"],
                         "result_pinned": v["result_pinned"], "equals_old_path": v["equal"]})
        del images, ref, variants
    if args.out:
        with open(args.out, "w", encoding="utf-8") as fh:
            fh.write("\n".join(json.dumps(l) for l in lines) + "\n")


if __name__ == "__main__":
    main()

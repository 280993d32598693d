"""Cost of FastFilmGrain's global-generator stream (VRGDG_GRAIN_NOISE=torch_cuda): the reference's loop on CUDA frames vs the node's
device path.

    python tools/global_stream_perf.py [--rounds 8] [--iters 10] [--warmup 3] [--out FILE]

Workloads (device-resident fp32 frames, intensity 0.04, saturation 0.5, batch_size 4, the node's default):
  grain_16x1080p_fp32  16 x 1920x1080
  grain_8x4K_fp32       8 x 3840x2160
Variants: "reference" (nodes.py:46-62 on CUDA frames: per mini-batch torch.randn_like from the global generator, the grain mix, the
multiply, add and clamp, then torch.cat), "node" (FastFilmGrain().apply_grain with VRGDG_GRAIN_NOISE=torch_cuda: two host calls for
the generator's increment, one vrgdg_grain_torch_global launch drawing the stream in the kernel).  Before timing, both run from the
same generator state and their outputs and the offsets they leave are compared.  Within each round the variants alternate (order
rotated every round), each timed with CUDA events over --iters back-to-back calls.  The card's name and power limit are read in the
same run."""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import natural_frames  # noqa: E402

PKG = "comfyui-vrgamedevgirl_b200"
I, SAT, BATCH = 0.04, 0.5, 4


def card():
    try:
        txt = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return {"nvidia-smi": txt}
    except Exception as e:  # noqa: BLE001
        return {"nvidia-smi": "unavailable: %s" % e}


def reference(images):
    """FastFilmGrain.apply_grain (nodes.py:46-62) with its device = the frames' CUDA device"""
    step = BATCH if BATCH > 0 else images.shape[0]
    chunks = []
    for i in range(0, images.shape[0], step):
        batch = images[i:i + step]
        g = torch.randn_like(batch)
        g[..., 0] *= 2.0
        g[..., 2] *= 3.0
        gray = g[..., 1].unsqueeze(-1).repeat(1, 1, 1, 3)
        mixed = SAT * g + (1.0 - SAT) * gray
        chunks.append((batch + mixed * I).clamp(0.0, 1.0))
    return torch.cat(chunks, dim=0)


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("global_stream_perf needs a CUDA device")
    os.environ["VRGDG_GRAIN_NOISE"] = "torch_cuda"
    pkg = importlib.import_module(PKG)
    node = pkg.FastFilmGrain()
    torch.cuda.init()
    gen = torch.cuda.default_generators[0]
    result = {"card": card(), "device": torch.cuda.get_device_name(0),
              "sms": torch.cuda.get_device_properties(0).multi_processor_count, "batch_size": BATCH, "workloads": {}}
    for name, (B, H, W) in {"grain_16x1080p_fp32": (16, 1080, 1920), "grain_8x4K_fp32": (8, 2160, 3840)}.items():
        x = natural_frames(B, H, W, seed=1).cuda()
        variants = {"reference": lambda: reference(x), "node": lambda: node.apply_grain(x, I, SAT, BATCH)[0]}
        torch.cuda.manual_seed(5)
        o0 = gen.get_offset()
        want = variants["reference"]()
        o_ref = gen.get_offset()
        gen.set_offset(o0)
        got = variants["node"]()
        same = torch.equal(got, want) and gen.get_offset() == o_ref
        del want, got
        for fn in variants.values():
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in variants}
        keys = list(variants)
        for r in range(args.rounds):
            for k in keys[r % len(keys):] + keys[:r % len(keys)]:
                times[k].append(timed(variants[k], args.iters))
        result["workloads"][name] = {
            "node_equals_reference": same,
            "ms_per_call": {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()},
            "gpx_per_s": {k: B * H * W / (statistics.median(v) * 1e-3) / 1e9 for k, v in times.items()},
        }
        del x
        torch.cuda.empty_cache()
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w", encoding="utf-8") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()

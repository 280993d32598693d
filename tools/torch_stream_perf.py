"""Cost of torch-stream grain (VRGDG_SEED_TORCH_PER_FRAME): this package's own generator vs torch's CUDA randn stream drawn in the
kernel vs the obvious alternative, torch.randn per frame materialised and fed to the exact ext_noise path.

    python tools/torch_stream_perf.py [--rounds 8] [--iters 10] [--warmup 3] [--out FILE]

Workloads (device-resident frames):
  grain_16x1080p_fp32   vrgdg_grain on 16 x 1920x1080 fp32 frames (intensity 0.05, saturation 0.4)
  unsharp_grain_8x4K_u8 unsharp 0.5 (zero border) + post grain on 8 x 3840x2160 uint8 BGR frames
Variants: "vrgdg" (the default generator, one Philox call per pixel pair), "torch_kernel" (the torch stream in the kernel: three
Philox calls and Box-Muller evaluations per pixel), "torch_randn" (one torch.randn of [H,W,3] per frame from a fresh seeded CUDA
generator, then the ext_noise path; for the uint8 workload the reference's byte path: bytes -> fp32 frames, the unsharp kernel, the
draws, vrgdg_grain, fp32 -> bytes).  Before timing, torch_kernel's output is compared with torch_randn's (must be equal).  Within
each round the variants alternate (order rotated every round), each timed with CUDA events over --iters back-to-back calls.  The
card's name and power limit are read in the same run."""
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
I, SAT, SEED, F0 = 0.05, 0.4, 31, 7


def card():
    try:
        txt = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return {"nvidia-smi": txt}
    except Exception as e:  # noqa: BLE001
        return {"nvidia-smi": "unavailable: %s" % e}


def per_frame_randn(B, H, W):
    return torch.stack([torch.randn([H, W, 3], generator=torch.Generator(device="cuda").manual_seed((SEED + F0 + i) & 0x7FFFFFFF),
                                    device="cuda") for i in range(B)])


def workloads(pkg):
    nv, ops, chain = pkg._native, pkg.ops, pkg.chain
    x = natural_frames(16, 1080, 1920, seed=1).cuda()
    grain = {
        "vrgdg": lambda: ops.grain(x, I, SAT, 1.0 - SAT, SEED, F0, nv.SEED_PER_FRAME),
        "torch_kernel": lambda: ops.grain(x, I, SAT, 1.0 - SAT, SEED, F0, nv.SEED_TORCH_PER_FRAME),
        "torch_randn": lambda: ops.grain(x, I, SAT, 1.0 - SAT, SEED, F0, nv.SEED_PER_FRAME, ext_noise=per_frame_randn(16, 1080, 1920)),
    }
    u8 = ops.rgb_to_u8bgr(natural_frames(8, 2160, 3840, seed=2).cuda())
    stencil = dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5, border=nv.BORDER_ZERO)
    post = dict(intensity=I, saturation_mix=SAT, seed=SEED)
    own = chain.PostChain(stencil=stencil, post_grain=dict(post, seed_mode=nv.SEED_PER_FRAME))
    tk = chain.PostChain(stencil=stencil, post_grain=dict(post, seed_mode=nv.SEED_TORCH_PER_FRAME))

    def materialised():
        sharp = ops.stencil3x3(ops.u8bgr_to_rgb(u8), nv.STENCIL_BOX_UNSHARP, 0.5, nv.BORDER_ZERO)     # the reference's fp32 frames
        return ops.rgb_to_u8bgr(ops.grain(sharp, I, SAT, 1.0 - SAT, SEED, F0, nv.SEED_PER_FRAME, ext_noise=per_frame_randn(8, 2160, 3840)))
    unsharp = {"vrgdg": lambda: own(u8, first_frame=F0), "torch_kernel": lambda: tk(u8, first_frame=F0), "torch_randn": materialised}
    return {"grain_16x1080p_fp32": (grain, 16 * 1080 * 1920), "unsharp_grain_8x4K_u8": (unsharp, 8 * 2160 * 3840)}


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
        raise SystemExit("torch_stream_perf needs a CUDA device")
    pkg = importlib.import_module(PKG)
    result = {"card": card(), "device": torch.cuda.get_device_name(0),
              "sms": torch.cuda.get_device_properties(0).multi_processor_count, "workloads": {}}
    for name, (variants, pixels) in workloads(pkg).items():
        same = torch.equal(variants["torch_kernel"](), variants["torch_randn"]())
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
            "torch_kernel_equals_torch_randn": same,
            "ms_per_call": {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()},
            "gpx_per_s": {k: pixels / (statistics.median(v) * 1e-3) / 1e9 for k, v in times.items()},
        }
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w", encoding="utf-8") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()

"""Cost of VRGDG_B200_PostChain's grain from the global CUDA generator (VRGDG_GRAIN_NOISE=torch_cuda): the fused node against the
four-node graph it replaces in that mode, against itself in the default mode, and the noise kernel alone against torch.randn_like.

    python tools/postchain_global_stream_perf.py [--rounds 6] [--iters 5] [--host-iters 1] [--warmup 2] [--out FILE]

Workloads (fp32 frames; grain 0.04 / saturation 0.5, colour match 1.0 to a 0.8-scaled first frame, 33^3 LUT at strength 10, unsharp
0.5 on the NumPy path, batch_size 4):
  16x1080p_fp32  16 x 1920x1080
  8x4K_fp32       8 x 3840x2160
Variants, each on CUDA frames ("cuda") and on pageable host frames ("host"):
  node_torch_cuda   VRGDG_B200_PostChain under torch_cuda: the noise of each upload chunk made by vrgdg_grain_noise_torch_global,
                    then the external-noise chain (vrgdg_chain_cm_apply, exact arithmetic)
  graph_torch_cuda  FastFilmGrain -> ColorMatchToReference -> VRGDG_LUTS -> FastUnsharpSharpen under torch_cuda
  node_default      VRGDG_B200_PostChain with this package's generator (CUDA frames only)
and, on CUDA frames, "noise_kernel" (ops.grain_noise_torch_global of the whole batch, one draw) against "randn_like" (torch.randn_like
of the same [B,H,W,3] fp32 tensor, which draws the same values).  Before timing, the node and the graph run from the same generator
state: their max |difference| and the offsets they leave are reported, and the noise kernel must equal randn_like.  Within each
round the variants of a group alternate (order rotated every round); device-resident variants are timed with CUDA events over
--iters back-to-back calls, host ones with a wall clock over --host-iters synchronised calls.  The card's name, power limit and SM
clock are read by nvidia-smi in the same run, before and after the timing."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import natural_frames  # noqa: E402

PKG = "comfyui-vrgamedevgirl_b200"
I, SAT, MATCH, LUT, LUT_STRENGTH, SHARP, BATCH = 0.04, 0.5, 1.0, "B200 Vintage 33.cube", 10.0, 0.5, 4
HBM_BYTES_PER_S = 3.35e12          # H100 SXM5 HBM3 peak


def card():
    try:
        txt = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return {"nvidia-smi name, power.limit, clocks.sm, clocks.max.sm": txt}
    except Exception as e:  # noqa: BLE001
        return {"nvidia-smi": "unavailable: %s" % e}


def timed_events(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def timed_wall(fn, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / iters


def run_group(variants, timer, iters, rounds, warmup):
    for fn in variants.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    keys = list(variants)
    for r in range(rounds):
        for k in keys[r % len(keys):] + keys[:r % len(keys)]:
            times[k].append(timer(variants[k], iters))
    return {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--host-iters", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("postchain_global_stream_perf needs a CUDA device")
    pkg = importlib.import_module(PKG)
    node, grain, cm, luts, sharp = (pkg.NODE_CLASS_MAPPINGS[k]() for k in
                                    ("VRGDG_B200_PostChain", "FastFilmGrain", "ColorMatchToReference", "VRGDG_LUTS", "FastUnsharpSharpen"))
    torch.cuda.init()
    gen = torch.cuda.default_generators[0]

    def with_noise(mode, fn):
        def call():
            os.environ["VRGDG_GRAIN_NOISE"] = mode
            return fn()
        return call

    result = {"card_before": card(), "device": torch.cuda.get_device_name(0), "sms": torch.cuda.get_device_properties(0).multi_processor_count,
              "batch_size": BATCH, "workloads": {}}
    for name, (B, H, W) in {"16x1080p_fp32": (16, 1080, 1920), "8x4K_fp32": (8, 2160, 3840)}.items():
        host = natural_frames(B, H, W, seed=1)
        ref = host[:1] * 0.8
        w = {}
        for where, x in (("cuda", host.cuda()), ("host", host)):
            r = ref.to(x.device)
            v = {"node_torch_cuda": with_noise("torch_cuda", lambda: node.apply_chain(x, I, SAT, MATCH, LUT, LUT_STRENGTH, "unsharp", SHARP,
                                                                                        False, BATCH, reference_image=r)[0]),
                 "graph_torch_cuda": with_noise("torch_cuda", lambda: sharp.apply_unsharp(luts.apply_lut(cm.match_color(
                     grain.apply_grain(x, I, SAT, BATCH)[0], r, MATCH, 1)[0], LUT, "auto", LUT_STRENGTH)[0], SHARP, False)[0])}
            torch.cuda.manual_seed(5)
            o0 = gen.get_offset()
            want = v["graph_torch_cuda"]()
            o_graph = gen.get_offset()
            gen.set_offset(o0)
            got = v["node_torch_cuda"]()
            w[where + "_node_vs_graph"] = {"max_abs_diff": float((got.cpu() - want.cpu()).abs().max()), "torch_equal": torch.equal(got, want),
                                           "offsets_equal": gen.get_offset() == o_graph}
            del want, got
            if where == "cuda":
                v["node_default"] = with_noise("vrgdg", lambda: node.apply_chain(x, I, SAT, MATCH, LUT, LUT_STRENGTH, "unsharp", SHARP,
                                                                                 False, BATCH, reference_image=r)[0])
                w["cuda_ms_per_call"] = run_group(v, timed_events, args.iters, args.rounds, args.warmup)
            else:
                w["host_ms_per_call"] = run_group(v, timed_wall, args.host_iters, args.rounds, 1)
        # the noise kernel alone: one draw of the whole batch
        x = host.cuda()
        seed = gen.initial_seed()
        o = gen.get_offset()
        kern = lambda: pkg.ops.grain_noise_torch_global(x, seed, o, 0, B, B)  # noqa: E731
        same = torch.equal(kern(), torch.randn_like(x))
        gen.set_offset(o)
        t = run_group({"noise_kernel": kern, "randn_like": lambda: torch.randn_like(x)}, timed_events, args.iters, args.rounds, args.warmup)
        nbytes = x.numel() * x.element_size()
        w["noise"] = {"kernel_equals_randn_like": same, "ms_per_call": t, "bytes_written": nbytes,
                      "share_of_3.35TB/s": {k: nbytes / (t[k]["median"] * 1e-3) / HBM_BYTES_PER_S for k in t}}
        w["gpx_per_s"] = {"%s_%s" % (g, k): B * H * W / (s["median"] * 1e-3) / 1e9
                          for g in ("cuda_ms_per_call", "host_ms_per_call") for k, s in w[g].items()}
        result["workloads"][name] = w
        del x, host
        torch.cuda.empty_cache()
    result["card_after"] = card()
    os.environ.pop("VRGDG_GRAIN_NOISE", None)
    text = json.dumps(result, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w", encoding="utf-8") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()

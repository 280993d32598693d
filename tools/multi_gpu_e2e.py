"""End to end through PostChain.run_host, pinned host frames -> pinned host frames, on 1, 2, ... N devices of one process.

    python tools/multi_gpu_e2e.py [--frames 32] [--repeats 3] [--steps 3] [--chunk 1]

Headline chain (bench.py's): grain -> colour match (one 4K reference) -> 33^3 LUT -> unsharp on 3840x2160 fp32 frames.  The same
host batch runs on the first k visible compute-capability-9.0 devices for every k (PostChain(devices=...), one host thread and one
PCIe link per device), plus two workers on device 0, which costs the sharded path's overhead and can gain nothing (one link).  The
device counts alternate within every repeat.  Each line: GPx/s, GB/s each way, the per-step times, and whether the result is
torch.equal to the one-device result.  Card names and power limits come from a read-only nvidia-smi query."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import natural_frames  # noqa: E402

PKG = "comfyui-vrgamedevgirl_b200"
H4K, W4K = 2160, 3840


def cards():
    q = "index,name,power.limit,clocks.max.sm,pci.bus_id"
    try:
        txt = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=60).stdout
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable: %s" % e
    return [dict(zip(q.split(","), (f.strip() for f in line.split(",")))) for line in txt.strip().splitlines()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=32, help="host batch (4K fp32 frames, 99.5 MB each), the same for every device count")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3, help="run_host calls per timing")
    ap.add_argument("--chunk", type=int, default=1, help="chunk_frames of run_host (bench.py's e2e leg uses 1)")
    args = ap.parse_args()
    pkg = importlib.import_module(PKG)
    nv = pkg._native
    devs = [torch.device("cuda", i) for i in range(torch.cuda.device_count()) if tuple(torch.cuda.get_device_capability(i)) == (9, 0)]
    if not devs:
        raise SystemExit("no visible device of compute capability 9.0")
    print(json.dumps({"cards": cards(), "visible_cc90": [torch.cuda.get_device_name(d) for d in devs],
                      "torch": torch.__version__, "cuda": torch.version.cuda}))

    base = natural_frames(4, H4K, W4K, seed=1)
    host_in = torch.empty((args.frames, H4K, W4K, 3), dtype=torch.float32, pin_memory=True)
    for i in range(args.frames):
        host_in[i].copy_(base[i % 4])
    ref = natural_frames(1, H4K, W4K, seed=4242)
    lut = pkg.VRGDG_LUTS._parse_cube_file(os.path.join(ROOT, PKG, "LUTS", "B200 Vintage 33.cube"))
    configs = [("1 device", devs[:1]), ("2 workers on device 0", [devs[0], devs[0]])]
    configs += [("%d devices" % k, devs[:k]) for k in range(2, len(devs) + 1)]
    chains = {name: pkg.chain.PostChain(grain=dict(intensity=0.04, saturation_mix=0.5, seed=42),
                                        colormatch=dict(reference_image=ref, strength=1.0), lut=dict(lut_data=lut, strength=10.0),
                                        stencil=dict(op=nv.STENCIL_BOX_UNSHARP, strength=0.5), devices=d) for name, d in configs}
    out = torch.empty_like(host_in, pin_memory=True)      # pinned once, reused by every call

    def run(name):
        return chains[name].run_host(host_in, chunk_frames=args.chunk, out=out)

    identical = {}
    for name, _ in configs:                     # warm-up (modules, allocator blocks, side streams of every worker) + output check
        run(name)
        if name == "1 device":
            want = out.clone()
        identical[name] = bool(torch.equal(out, want))
    del want
    times = {name: [] for name, _ in configs}
    for _ in range(args.repeats):
        for name, _ in configs:                 # device counts alternate within every repeat
            t0 = time.perf_counter()
            for _ in range(args.steps):
                run(name)                       # returns once the last download has landed in host memory
            times[name].append((time.perf_counter() - t0) / args.steps)
    px = args.frames * H4K * W4K
    nbytes = host_in.numel() * host_in.element_size()
    one = sorted(times["1 device"])[len(times["1 device"]) // 2]
    for name, d in configs:
        med = sorted(times[name])[len(times[name]) // 2]
        line = {"config": name, "devices": [x.index for x in d], "frames": args.frames, "chunk_frames": args.chunk,
                "gpx_s": round(px / med / 1e9, 3), "gb_s_each_way": round(nbytes / med / 1e9, 2),
                "ms_per_call": [round(t * 1e3, 1) for t in times[name]], "bit_identical_to_1_device": identical[name]}
        if len(set(d)) > 1:                     # a speed-up only means something over distinct cards
            line["speedup_vs_1_device"] = round(one / med, 3)
        print(json.dumps(line))


if __name__ == "__main__":
    main()

"""The unchanged four-node workflow FastFilmGrain -> ColorMatchToReference -> VRGDG_LUTS -> FastUnsharpSharpen on pageable host
frames, with VRGDG_DEVICES naming 1, 2, ... N devices of one process.

    python tools/multi_gpu_stock_nodes.py [--frames 16] [--repeats 3] [--steps 2]

3840x2160 fp32 frames in pageable host memory (what a ComfyUI IMAGE batch is), one 4K reference frame, the widgets bench.py's
stock-node leg uses.  Configurations: VRGDG_DEVICES unset (one device), the first k visible compute-capability-9.0 devices for every
k >= 2 (VRGDG_DEVICES=i,j,...), and two workers on device 0 (handed to the node modules directly: the parser rejects a repeated
index), which costs the sharded path's overhead over one PCIe link and can gain nothing.  The configurations alternate within every
repeat.  Each line: GPx/s, the per-step times, and whether the result is torch.equal to the one-device result.  Card names and power
limits come from a read-only nvidia-smi query."""
import argparse
import importlib
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from helpers import natural_frames  # noqa: E402
from multi_gpu_e2e import cards  # noqa: E402

PKG = "comfyui-vrgamedevgirl_b200"
H4K, W4K = 2160, 3840
LUT = "B200 Vintage 33.cube"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16, help="pageable host batch (4K fp32 frames, 99.5 MB each), the same for every configuration")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2, help="workflow runs per timing")
    args = ap.parse_args()
    pkg = importlib.import_module(PKG)
    modules = [importlib.import_module(PKG + "." + m) for m in ("filter_nodes", "lut_nodes", "chain_nodes")]
    from_env = modules[0].devices_from_env
    devs = [torch.device("cuda", i) for i in range(torch.cuda.device_count()) if tuple(torch.cuda.get_device_capability(i)) == (9, 0)]
    if not devs:
        raise SystemExit("no visible device of compute capability 9.0")
    print(json.dumps({"cards": cards(), "visible_cc90": [torch.cuda.get_device_name(d) for d in devs],
                      "torch": torch.__version__, "cuda": torch.version.cuda}))

    base = natural_frames(4, H4K, W4K, seed=1)
    host_in = torch.empty((args.frames, H4K, W4K, 3), dtype=torch.float32)          # pageable
    for i in range(args.frames):
        host_in[i].copy_(base[i % 4])
    ref = natural_frames(1, H4K, W4K, seed=4242)
    nodes = (pkg.FastFilmGrain(), pkg.ColorMatchToReference(), pkg.VRGDG_LUTS(), pkg.FastUnsharpSharpen())
    # name -> (VRGDG_DEVICES value or None, device list handed to the node modules or None)
    configs = {"1 device": (None, None), "2 workers on device 0": (None, [devs[0], devs[0]])}
    configs.update({"%d devices" % k: (",".join(str(d.index) for d in devs[:k]), None) for k in range(2, len(devs) + 1)})

    def select(name):
        env, workers = configs[name]
        if env is None:
            os.environ.pop("VRGDG_DEVICES", None)
        else:
            os.environ["VRGDG_DEVICES"] = env
        for m in modules:
            m.devices_from_env = from_env if workers is None else (lambda: list(workers))

    def step():
        torch.manual_seed(0)                    # the grain node draws its seed from torch's generator
        a = nodes[0].apply_grain(host_in, 0.04, 0.5, 4)[0]
        b = nodes[1].match_color(a, ref, 1.0, 1)[0]
        c = nodes[2].apply_lut(b, LUT, "auto", 10.0)[0]
        return nodes[3].apply_unsharp(c, 0.5, False)[0]       # host tensors: every node returns once its last download has landed

    identical, want = {}, None
    try:
        for name in configs:                    # warm-up (modules, pinned blocks, side streams of every worker) + output check
            select(name)
            got = step()
            if want is None:
                want = got
            identical[name] = bool(torch.equal(got, want))
        del want, got
        times = {name: [] for name in configs}
        for _ in range(args.repeats):
            for name in configs:                # configurations alternate within every repeat
                select(name)
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    step()
                times[name].append((time.perf_counter() - t0) / args.steps)
    finally:
        select("1 device")
    px = args.frames * H4K * W4K
    one = sorted(times["1 device"])[len(times["1 device"]) // 2]
    for name, (env, workers) in configs.items():
        med = sorted(times[name])[len(times[name]) // 2]
        line = {"config": name, "VRGDG_DEVICES": env, "frames": args.frames, "gpx_s": round(px / med / 1e9, 3),
                "ms_per_step": [round(t * 1e3, 1) for t in times[name]], "bit_identical_to_1_device": identical[name]}
        if workers is not None:
            line["workers"] = [str(d) for d in workers]
        if env is not None:                     # a speed-up only means something over distinct cards
            line["speedup_vs_1_device"] = round(one / med, 3)
        print(json.dumps(line))


if __name__ == "__main__":
    main()

"""VRGDG_B200_HistogramColorMatch against a reference clip (n_ref == B) versus the loop a user needs without it.

    python tools/hist_reference_clip_perf.py [--batch-size 8] [--rounds 5] [--out FILE]

Workloads: 16 x 1920x1080 and 8 x 3840x2160 fp32 frames, each against a reference clip of as many frames of the same size, from CUDA
frames (reference clip on the card) and from pageable host frames (reference clip on the host, host result).
Variants:
  clip        one node call with the B-frame reference clip: each chunk uploads its own reference frames and makes one
              vrgdg_histmatch_apply_refs call.
  frame_loop  B node calls, one per frame, each with its one reference frame, and the results concatenated where they land.
The variants alternate within every round (order flipped every other round) after one warm-up round that is not reported.  Per
variant: median / min / max wall time of a call (each ends with a device synchronise; host results are on the host), the peak growth
of torch.cuda.max_memory_allocated during the call against the reference clip's bytes, and whether the two outputs are torch.equal.
The card's name and power limit are printed in the same run."""
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
WORKLOADS = {"16x1080p_fp32": (16, 1080, 1920), "8x4K_fp32": (8, 2160, 3840)}
STRENGTH = 0.8


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-size", type=int, default=8, help="the node's batch_size widget (frames per chunk)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has nothing to report without one")
    os.environ.pop("VRGDG_DEVICES", None)
    pkg = importlib.import_module(PKG)
    dev = torch.device("cuda", 0)
    lines = []
    emit(lines, {"card": card(), "device": torch.cuda.get_device_name(dev), "torch": torch.__version__, "cuda": torch.version.cuda})
    node = pkg.NODE_CLASS_MAPPINGS["VRGDG_B200_HistogramColorMatch"]()
    bs = args.batch_size
    cpu = torch.Generator().manual_seed(5)
    for name, (n, h, w) in WORKLOADS.items():
        frames_host = torch.rand(n, h, w, 3, generator=cpu)
        refs_host = torch.rand(n, h, w, 3, generator=cpu) * 0.6 + 0.2
        for where in ("cuda", "host"):
            images = frames_host if where == "host" else frames_host.to(dev)
            refs = refs_host if where == "host" else refs_host.to(dev)
            variants = {"clip": lambda: node.match_histogram(images, refs, STRENGTH, bs)[0],
                        "frame_loop": lambda: torch.cat([node.match_histogram(images[i:i + 1], refs[i:i + 1], STRENGTH, bs)[0]
                                                         for i in range(n)])}

            def run(k):
                torch.cuda.synchronize(dev)
                torch.cuda.reset_peak_memory_stats(dev)
                base = torch.cuda.memory_allocated(dev)
                t0 = time.perf_counter()
                out = variants[k]()
                torch.cuda.synchronize(dev)
                return out, time.perf_counter() - t0, torch.cuda.max_memory_allocated(dev) - base
            res = {k: {"s": [], "peak": 0} for k in variants}
            equal = True
            for r in range(args.rounds + 1):                   # round 0 warms both paths up and is not reported
                outs = {}
                for k in (list(variants) if r % 2 == 0 else list(reversed(list(variants)))):
                    outs[k], dt, peak = run(k)
                    if r > 0:
                        res[k]["s"].append(dt)
                        res[k]["peak"] = max(res[k]["peak"], peak)
                equal = equal and bool(torch.equal(outs["clip"], outs["frame_loop"]))
                del outs
            clip = refs.numel() * refs.element_size()
            for k, v in res.items():
                med = statistics.median(v["s"])
                emit(lines, {"workload": "%s_%s" % (name, where), "variant": k, "batch_size": bs, "rounds": args.rounds,
                             "ms_per_call_median": round(med * 1e3, 2), "ms_min": round(min(v["s"]) * 1e3, 2),
                             "ms_max": round(max(v["s"]) * 1e3, 2), "peak_device_bytes": v["peak"], "reference_clip_bytes": clip,
                             "peak_over_clip": round(v["peak"] / clip, 3), "clip_equals_frame_loop": equal})
            del images, refs, variants
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w", encoding="utf-8") as fh:
            fh.write("\n".join(json.dumps(l) for l in lines) + "\n")


if __name__ == "__main__":
    main()

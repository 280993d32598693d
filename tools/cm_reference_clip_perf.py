"""ColorMatchToReference against a reference clip (n_ref == B): the whole-clip path the package ran before against the streamed one.

    python tools/cm_reference_clip_perf.py [--frames 32] [--batch-size 4] [--rounds 3] [--out FILE]

Workloads: --frames 3840x2160 fp32 frames against a reference clip of as many 3840x2160 frames, and against one of 1920x1080 frames;
each from host frames (pageable, host result, reference clip on the host) and from CUDA frames (reference clip on the card).
Variants:
  whole_clip  the node as it was: the whole reference clip uploaded and converted at once, vrgdg_lab_moments over all of it before the
              first frame, then the frames streamed with one vrgdg_chain_cm_apply per chunk on the per-frame sums of its indices.
  streamed    the node now: each chunk uploads only the reference frames of its indices and makes one vrgdg_chain_cm_apply_refs call.
The variants alternate within every round (order flipped every other round) after one warm-up round that is not reported.  Per
variant: median / min / max wall time of a call (each ends with a device synchronise; host results are on the host), the peak growth
of torch.cuda.max_memory_allocated during the call, and whether its output is torch.equal to the whole-clip path's.  The card's name
and power limit are printed in the same run."""
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
H, W = 2160, 3840
REF_SIZES = {"ref_4K": (2160, 3840), "ref_1080p": (1080, 1920)}
STRENGTH = 0.8


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        txt = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=60).stdout
    except (OSError, subprocess.SubprocessError) as e:
        return {"nvidia-smi": "unavailable: %s" % e}
    return dict(zip(q.split(","), (f.strip() for f in txt.strip().split(","))))


def whole_clip(pkg, rt, images, reference_image, t, batch_size):
    """ColorMatchToReference.match_color with n_ref == B as the package ran it before the reference clip was streamed"""
    nv, ops = pkg._native, pkg.ops
    dev = rt.compute_device(images)
    with torch.cuda.device(dev):
        ref_sums = ops.lab_moments(rt.upload(reference_image, dev).to(images.dtype))
    d = nv.ChainDesc()
    d.colormatch_enabled, d.cm_t, d.cm_one_minus_t = 1, t, 1.0 - t

    def make_fn(c):
        sums = ref_sums.to(c)
        state = {"scratch": None}

        def run(frames, first):
            out, state["scratch"] = ops.chain_cm_apply(frames, d, sums[first:first + frames.shape[0]], scratch=state["scratch"])
            return out
        return run
    return rt.run_frames(images, make_fn, batch_size, rt.result_device(images), dev, None)


def emit(lines, line):
    lines.append(line)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--batch-size", type=int, default=4, help="the node's batch_size widget (frames per chunk)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON lines here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU and has nothing to report without one")
    os.environ.pop("VRGDG_DEVICES", None)
    pkg = importlib.import_module(PKG)
    rt = importlib.import_module(PKG + "._runtime")
    dev = torch.device("cuda", 0)
    lines = []
    emit(lines, {"card": card(), "device": torch.cuda.get_device_name(dev), "torch": torch.__version__, "cuda": torch.version.cuda})
    node = pkg.ColorMatchToReference()
    n, bs = args.frames, args.batch_size
    cpu = torch.Generator().manual_seed(5)
    frames_host = torch.rand(n, H, W, 3, generator=cpu)
    for ref_name, (rh, rw) in REF_SIZES.items():
        refs_host = torch.rand(n, rh, rw, 3, generator=cpu) * 0.8 + 0.1
        for where in ("host", "cuda"):
            images = frames_host if where == "host" else frames_host.to(dev)
            refs = refs_host if where == "host" else refs_host.to(dev)
            variants = {"whole_clip": lambda: whole_clip(pkg, rt, images, refs, STRENGTH, bs),
                        "streamed": lambda: node.match_color(images, refs, STRENGTH, bs)[0]}

            def run(k):
                torch.cuda.synchronize(dev)
                torch.cuda.reset_peak_memory_stats(dev)
                base = torch.cuda.memory_allocated(dev)
                t0 = time.perf_counter()
                out = variants[k]()
                torch.cuda.synchronize(dev)
                return out, time.perf_counter() - t0, torch.cuda.max_memory_allocated(dev) - base
            res = {k: {"s": [], "peak": 0} for k in variants}
            equal = None
            for r in range(args.rounds + 1):                   # round 0 warms both paths up and is not reported
                outs = {}
                for k in (list(variants) if r % 2 == 0 else list(reversed(list(variants)))):
                    outs[k], dt, peak = run(k)
                    if r > 0:
                        res[k]["s"].append(dt)
                        res[k]["peak"] = max(res[k]["peak"], peak)
                if r == 0:
                    equal = bool(torch.equal(outs["streamed"], outs["whole_clip"]))
                del outs
            clip = refs.numel() * refs.element_size()
            for k, v in res.items():
                med = statistics.median(v["s"])
                emit(lines, {"workload": "%dx4K_fp32_frames_%s_%s" % (n, ref_name, where), "variant": k, "batch_size": bs,
                             "ms_per_call_median": round(med * 1e3, 1), "ms_min": round(min(v["s"]) * 1e3, 1),
                             "ms_max": round(max(v["s"]) * 1e3, 1), "peak_device_bytes": v["peak"],
                             "reference_clip_bytes": clip, "streamed_equals_whole_clip": equal})
            del images, refs, variants
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w", encoding="utf-8") as fh:
            fh.write("\n".join(json.dumps(l) for l in lines) + "\n")


if __name__ == "__main__":
    main()

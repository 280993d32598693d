"""The RGBA stencil matrix: which (dtype, op, border, shape) cases tests/test_gpu_rgba_stencil.py runs against the oracle, and a
parser of vrgdg_inst.cuh's launch_tile_rgba naming the (dtype, op, exact) kernel paths it can select.  No GPU and no torch needed
here, so the CPU suite can check that the cases reach every path (tests/test_rgba_stencil_cpu.py)."""
import itertools
import os
import re
from collections import namedtuple

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INST = os.path.join(ROOT, "comfyui-vrgamedevgirl_b200", "csrc", "vrgdg_inst.cuh")

DTYPES = ("f32", "f16", "bf16")
ULP = {"f16": 2.0 ** -11, "bf16": 2.0 ** -8}                        # spacing of the 16-bit type in [0.5, 1)
BOX_UNSHARP, LAPLACIAN_CPU, LAPLACIAN_GPU, SOBEL_CPU, SOBEL_GPU = 1, 2, 3, 4, 5
REPLICATE, ZERO = 0, 1
RGBA_OPS = (BOX_UNSHARP, LAPLACIAN_CPU, SOBEL_CPU)                  # the ops vrgdg_stencil3x3_ch takes on 4 channels
# (op, border) pairs with a reference function: the NumPy paths (edge replicated) and the avg_pool2d unsharp (zero padded)
PAIRS = ((BOX_UNSHARP, REPLICATE), (BOX_UNSHARP, ZERO), (LAPLACIAN_CPU, REPLICATE), (SOBEL_CPU, REPLICATE))
STRENGTH = {BOX_UNSHARP: 0.7, LAPLACIAN_CPU: 0.3, SOBEL_CPU: 0.25}
SHAPES = {"tma": (2, 70, 136),       # 3 x 3 tiles (544-element rows: 240 + 240 + 64; 70 rows: 32 + 32 + 6), rows 16-byte aligned
          "ragged": (2, 41, 75),     # odd W, under VRGDG_NO_TMA=1: the generic loader
          "small": (3, 9, 11)}       # smaller than one 34 x 256 box: the generic loader without forcing it
PATH = {"tma": "tma", "ragged": "generic", "small": "generic"}

Case = namedtuple("Case", "dtype op border shape")
CASES = [Case(d, op, b, s) for d, (op, b), s in itertools.product(DTYPES, PAIRS, SHAPES)]


def exact(dtype):
    """exact stencil arithmetic on fp32 frames, the fast variant on 16-bit ones (vrgdg_stencil3x3_ch)"""
    return dtype == "f32"


def kernel_of(case):
    return (case.dtype, case.op, exact(case.dtype))


def instantiated(path=INST):
    """{(dtype, op, EXACT)} launch_tile_rgba can run: the ops of its `case` labels that reach a launch_tile_k<T, 0, EXACT, 4> call,
    with the calls under `sizeof(T) == 4` for fp32 and the others for the 16-bit types (uint8 returns before the switch)."""
    with open(path, encoding="utf-8") as fh:
        src = fh.read()
    m = re.search(r"cudaError_t launch_tile_rgba\(.*?switch \(Q\.op\) \{(.*?)\n    \}", src, re.S)
    assert m, "no switch in launch_tile_rgba"
    out = set()
    for labels, block in re.findall(r"((?:case \d+:\s*)+)(.*?)(?=case \d+:|default:)", m.group(1), re.S):
        ops = [int(v) for v in re.findall(r"case (\d+):", labels)]
        assert "if constexpr (sizeof(T) == 4)" in block, "launch_tile_rgba no longer splits fp32 from the 16-bit types"
        f32, _, half = block.partition("} else {")
        for part, dts in ((f32, ("f32",)), (half, ("f16", "bf16"))):
            for ex in re.findall(r"launch_tile_k<T, 0, (true|false), 4>", part):
                for op in ops:
                    for dt in dts:
                        out.add((dt, op, ex == "true"))
    return out

"""The RGBA post-chain matrix: which (dtype, stages, op, border, LUT, blend, shape) cases tests/test_gpu_rgba_chain.py runs against
the oracle, and a parser of vrgdg_inst.cuh's launch_tile_rgba_lut naming the (dtype, op, exact stencil) kernel paths it can select.
No GPU and no torch needed here, so the CPU suite can check that the cases reach every path (tests/test_rgba_chain_cpu.py)."""
import itertools
import os
import re
from collections import namedtuple

import rgba_stencil_matrix as rsm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INST = os.path.join(ROOT, "comfyui-vrgamedevgirl_b200", "csrc", "vrgdg_inst.cuh")

DTYPES = rsm.DTYPES
ULP = rsm.ULP
PAIRS = rsm.PAIRS                  # (op, border) pairs with a reference function on RGBA
STRENGTH = rsm.STRENGTH
SHAPES = rsm.SHAPES                # TMA, ragged under VRGDG_NO_TMA=1, smaller than one box
PATH = rsm.PATH
# the shipped 33^3 table, a non-unit DOMAIN_MIN / DOMAIN_MAX, and a generated 65^3 table (helpers.write_big_cube)
LUTS = {"vintage33": os.path.join(ROOT, "comfyui-vrgamedevgirl_b200", "LUTS", "B200 Vintage 33.cube"),
        "domain5": os.path.join(ROOT, "tests", "golden", "domain_5.cube"),
        "big65": None}
BIG_LUT_SIZE = 65
LUT_STRENGTHS = (10.0, 3.5)        # blend 1 (alpha copied) and 0.35 (alpha blended with itself)
STAGES = ("lut", "stencil", "both")

Case = namedtuple("Case", "dtype stages op border lut strength shape")
CASES = ([Case(d, "both", op, b, lut, s, sh) for d, (op, b), lut, s, sh in itertools.product(DTYPES, PAIRS, LUTS, LUT_STRENGTHS, SHAPES)]
         + [Case(d, "lut", None, None, lut, s, sh) for d, lut, s, sh in itertools.product(DTYPES, LUTS, LUT_STRENGTHS, SHAPES)]
         + [Case(d, "stencil", op, b, None, None, sh) for d, (op, b), sh in itertools.product(DTYPES, PAIRS, SHAPES)])


def case_id(c):
    parts = [c.dtype, c.stages]
    if c.op is not None:
        parts.append("op%d-border%d" % (c.op, c.border))
    if c.lut is not None:
        parts.append("%s-s%g" % (c.lut, c.strength))
    return "-".join(parts + [c.shape])


def exact(dtype):
    """exact stencil arithmetic on fp32 frames, the fast variant on 16-bit ones (the 3-channel chain's rule)"""
    return dtype == "f32"


def kernel_of(case):
    """the launch_tile_rgba_lut path of a case, or None when the case runs another kernel (LUT alone: k_lut_rgba; stencil alone:
    launch_tile_rgba)"""
    return (case.dtype, case.op, exact(case.dtype)) if case.stages == "both" else None


def instantiated(path=INST):
    """{(dtype, op, exact stencil)} launch_tile_rgba_lut can run: the ops of its `case` labels that reach a launch_tile_k<T, ST_LUT,
    EXACT, 4> call, guarded by `if (Q.exact_stencil)` or `if (!Q.exact_stencil)`, with the calls under `sizeof(T) == 4` for fp32
    and the others for the 16-bit types (uint8 returns before the switch)."""
    with open(path, encoding="utf-8") as fh:
        src = fh.read()
    m = re.search(r"cudaError_t launch_tile_rgba_lut\(.*?switch \(Q\.op\) \{(.*?)\n    \}", src, re.S)
    assert m, "no switch in launch_tile_rgba_lut"
    out = set()
    for labels, block in re.findall(r"((?:case \d+:\s*)+)(.*?)(?=case \d+:|default:)", m.group(1), re.S):
        ops = [int(v) for v in re.findall(r"case (\d+):", labels)]
        assert "if constexpr (sizeof(T) == 4)" in block, "launch_tile_rgba_lut no longer splits fp32 from the 16-bit types"
        f32, _, half = block.partition("} else {")
        for part, dts in ((f32, ("f32",)), (half, ("f16", "bf16"))):
            for neg, lut_exact in re.findall(r"if \((!?)Q\.exact_stencil\) return launch_tile_k<T, ST_LUT, (true|false), 4>", part):
                assert lut_exact == "true", "the RGBA chain's LUT is the exact one of the 3-channel chain"
                for op in ops:
                    for dt in dts:
                        out.add((dt, op, neg != "!"))
    return out

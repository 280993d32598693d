"""The fused-chain matrix: which stage combinations, frame dtypes, noise sources, colour-match schedules and shapes
tests/test_gpu_chain_matrix.py runs against oracle.chain_compose, the documented error bar of each case, and a mirror of how
vrgdg_abi.cu picks the kernel for a case.  No GPU and no torch needed here, so the CPU suite can check that the matrix reaches
every k_tile / k_point instantiation (tests/test_chain_matrix_coverage.py)."""
import itertools
import os
import re
from collections import namedtuple

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INST = os.path.join(ROOT, "comfyui-vrgamedevgirl_b200", "csrc", "vrgdg_inst.cuh")

ST_GRAIN, ST_CM, ST_LUT, ST_POST, ST_CMF = 1, 2, 4, 8, 16          # vrgdg_kernels.cuh
DTYPES = ("f32", "f16", "bf16", "u8")
ULP = {"f16": 2.0 ** -11, "bf16": 2.0 ** -8}                        # spacing of the 16-bit type in [0.5, 1)

UNSHARP_REPLICATE = (1, 0)
# (op, border) pairs the oracle has a reference function for (oracle.CHAIN_STENCILS); the other pairs (e.g. a NumPy-path op with
# zero borders) are not reference behaviour and stay outside the matrix
STENCIL_PAIRS = ((1, 0), (1, 1), (2, 0), (3, 1), (4, 0), (5, 1))
STENCIL_STRENGTH = {1: 0.5, 2: 0.3, 3: 0.3, 4: 0.25, 5: 0.25}

# noise of the first grain stage: the external N(0,1) tensor in exact or fast arithmetic, or the in-kernel generator in either
# seed mode.  Post grain always draws from the generator.
NOISES = ("ext", "ext_fast", "clip", "frame")
# colour-match schedules: one vrgdg_chain_cm_apply call (f-planes on fp32 with W % 4 == 0; pipelined when there is a LUT and more
# than one group), the recompute schedule, groups one after the other, the three-call path, and 1- or 2-frame groups
SCHEDULES = ("default", "recompute", "serial", "split", "g1", "g2")
SHAPES = {"tma": (2, 72, 176),       # 3 x 3 tiles of every dtype (ragged last row and column), seams inside the frame, rows
                                     # 16-byte aligned for every dtype
          "ragged": (3, 37, 53),     # W % 4 != 0: generic loader, scalar k_point, no f-planes
          "notma": (2, 72, 176),     # the TMA shape under VRGDG_NO_TMA=1
          "groups": (5, 72, 176)}    # colour-match schedules: 5 frames in 1- or 2-frame groups wrap the double buffers

Case = namedtuple("Case", "grain cm lut post stencil dtype noise schedule shape")


def _stage_sets():
    """(grain, cm, lut, post, stencil): every subset of {grain, colour match, LUT, post grain} x {no stencil, unsharp-replicate},
    then every (op, border) pair behind grain + LUT and behind grain + colour match + LUT."""
    out = []
    for g, c, l, p in itertools.product((0, 1), repeat=4):
        for st in (None, UNSHARP_REPLICATE):
            if g or c or l or p or st:
                out.append((g, c, l, p, st))
    for g, c, l in ((1, 0, 1), (1, 1, 1)):
        for st in STENCIL_PAIRS:
            if st != UNSHARP_REPLICATE:
                out.append((g, c, l, 0, st))
    return out


STAGE_SETS = _stage_sets()


def _noises(grain, choice=NOISES):
    return choice if grain else ("none",)


def build_cases():
    cases = []
    for (g, c, l, p, st), dt in itertools.product(STAGE_SETS, DTYPES):
        for nz in _noises(g):
            cases.append(Case(g, c, l, p, st, dt, nz, "default", "tma"))
        # the generic loader: exact arithmetic and the generator on the ragged shape, the generator (as production runs) on the
        # TMA shape, so that both EXACT variants of every grain kernel meet the generic loader
        for nz in _noises(g, ("ext", "clip")):
            cases.append(Case(g, c, l, p, st, dt, nz, "default", "ragged"))
        cases.append(Case(g, c, l, p, st, dt, "clip" if g else "none", "default", "notma"))
        if c and st in (None, UNSHARP_REPLICATE):
            for nz in _noises(g, ("ext", "frame")):
                for sch in SCHEDULES:
                    cases.append(Case(g, c, l, p, st, dt, nz, sch, "groups"))
    return cases


CASES = build_cases()


def case_id(c):
    stages = "+".join(n for n, on in (("grain", c.grain), ("cm", c.cm), ("lut", c.lut)) if on) or "none"
    st = "st%d%s" % (c.stencil[0], "z" if c.stencil[1] else "r") if c.stencil else "nost"
    return "-".join([stages, st, "post" if c.post else "nopost", c.dtype, c.noise, c.schedule, c.shape])


def shape_of(c):
    return SHAPES[c.shape]


# ---- error bars -----------------------------------------------------------------------------------------------------------
# max |kernel - oracle.chain_compose| per case (fp32 oracle; 16-bit kernels are compared after up-casting, uint8 as bytes):
#   fp32, external noise, exact, NumPy-path op or unsharp-zero (or none), no colour match   0 (torch.equal)
#   torch-path ops 3 (Laplacian GPU) and 5 (Sobel GPU): conv2d has no defined summation order  1e-5
#   fp32 fast arithmetic or in-kernel noise (FMA-contracted blends, coefficient LUT cells)   4e-6
#   any chain with colour match (kornia Lab in fp32 vs fp64 statistics, then the inverse)     1e-5
#   post grain (FMA blend of the post-grain noise)                                             + 1e-6 on the bar above
#   fp16 / bf16: one spacing of the type in [0.5, 1) (2^-11 / 2^-8)                           + 1e-5 with colour match, + 1e-6 with post grain
#   uint8: bytes equal when the fp32 bar is 0; otherwise |delta| <= 1 code on < 1e-3 of the bytes (truncating clip(x*255) turns
#          any difference next to an integer into a whole code)
BAR_TORCH_OP, BAR_FAST, BAR_CM, BAR_POST = 1e-5, 4e-6, 1e-5, 1e-6
U8_FLIP_FRACTION = 1e-3


def fast_first_stage(c):
    return bool(c.grain) and c.noise in ("ext_fast", "clip", "frame")


def float_bar(c):
    """max |delta| of fp32 frames against the oracle; 0 means torch.equal"""
    bar = 0.0
    if c.stencil and c.stencil[0] in (3, 5):
        bar = BAR_TORCH_OP
    if fast_first_stage(c):
        bar = max(bar, BAR_FAST)
    if c.cm:
        bar = max(bar, BAR_CM)
    if c.post:
        bar += BAR_POST
    return bar


def half_bar(c):
    return ULP[c.dtype] + (BAR_CM if c.cm else 0.0) + (BAR_POST if c.post else 0.0)


# ---- mirror of the kernel choice (chain_apply_core / vrgdg_chain_cm_apply / chain_point_params) ------------------------------
def uses_fplanes(c):
    """cm_uses_planes: fp32 frames with W % 4 == 0 on the one-call schedules other than recompute (torch allocations are aligned)"""
    W = shape_of(c)[2]
    return bool(c.cm) and c.schedule not in ("split", "recompute") and c.dtype == "f32" and W % 4 == 0


def kernel_of(c):
    """(kernel, dtype, mask, EXACT) of the apply pass of a case, or None when nothing runs (not in the matrix)."""
    mask = (ST_GRAIN if c.grain else 0) | (ST_CM if c.cm else 0) | (ST_LUT if c.lut else 0)
    exact = not fast_first_stage(c)                          # chain_point_params
    if uses_fplanes(c):
        mask = (mask & ST_LUT) | ST_CMF
    if not (c.stencil or c.post):
        if mask == 0:
            return None
        kernel = "point"
    else:
        kernel = "tile"
        if c.post and mask == 0:
            mask = ST_POST
    # only masks with grain (or with the f-plane colour match feeding a LUT) have an inexact instantiation
    has_inexact = bool(mask & ST_GRAIN) or mask == (ST_CMF | ST_LUT)
    return (kernel, c.dtype, mask, exact if has_inexact else True)


def exact_stencil(c):
    """Q.exact_stencil: the NumPy evaluation order is kept for exact chains on fp32 and byte frames"""
    return not fast_first_stage(c) and c.dtype in ("f32", "u8")


# ---- what vrgdg_inst.cuh instantiates --------------------------------------------------------------------------------------
_NAMES = {"ST_GRAIN": ST_GRAIN, "ST_CM": ST_CM, "ST_LUT": ST_LUT, "ST_POST": ST_POST, "ST_CMF": ST_CMF}


def _mask_value(expr):
    expr = expr.strip()
    if re.fullmatch(r"\d+", expr):
        return int(expr)
    v = 0
    for name in expr.split("|"):
        v |= _NAMES[name.strip()]
    return v


def instantiated(path=INST):
    """{(kernel, dtype, mask, EXACT)} from the switch statements of launch_point / launch_tile: VRGDG_PT(M) / VRGDG_TL(M) give
    EXACT = true, and false too when M has ST_GRAIN; explicit `case` labels give what their launch_*<T, M, EXACT> calls name, for fp32
    only when guarded by sizeof(T) == 4."""
    with open(path, encoding="utf-8") as fh:
        src = fh.read()
    out = set()
    for kernel, fn, macro, callee in (("point", "launch_point", "VRGDG_PT", "launch_point_v"), ("tile", "launch_tile", "VRGDG_TL", "launch_tile_k")):
        m = re.search(r"cudaError_t %s\(.*?switch \(mask\) \{(.*?)\n  \}" % fn, src, re.S)
        assert m, "no switch in %s" % fn
        body = m.group(1)
        for mv in re.findall(r"%s\((\d+)\)" % macro, body):
            mv = int(mv)
            for dt in DTYPES:
                out.add((kernel, dt, mv, True))
                if mv & ST_GRAIN:
                    out.add((kernel, dt, mv, False))
        for label, block in re.findall(r"case ([A-Z_ |0-9]+):(.*?)(?=\n    case |\n    default:)", body, re.S):
            mv = _mask_value(label)
            dts = ("f32",) if "sizeof(T) == 4" in block else DTYPES
            for ex in re.findall(r"%s<T, [^,>]+, (true|false)>" % callee, block):
                for dt in dts:
                    out.add((kernel, dt, mv, ex == "true"))
    return out

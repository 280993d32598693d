"""CPU guard of the fused-chain matrix (tests/test_gpu_chain_matrix.py): every k_point / k_tile instantiation that
vrgdg_inst.cuh's launch_point / launch_tile can select is reached by at least one matrix case, for every frame dtype it is built for.
A kernel path added without a matrix case fails here, without a GPU."""
import chain_matrix as cmx


def test_instantiations_are_parsed():
    inst = cmx.instantiated()
    # anchors: the plain stencil, the enhancer chain, the f-plane colour match (fp32 only), an inexact grain chain
    for k in (("tile", "u8", 0, True), ("tile", "bf16", cmx.ST_POST, True), ("tile", "f32", cmx.ST_CMF, True),
              ("point", "f32", cmx.ST_CMF | cmx.ST_LUT, False), ("tile", "f16", cmx.ST_GRAIN | cmx.ST_CM | cmx.ST_LUT, False)):
        assert k in inst, k
    assert ("tile", "f16", cmx.ST_CMF, True) not in inst and ("point", "f32", cmx.ST_LUT, False) not in inst
    assert ("point", "f32", cmx.ST_POST, True) not in inst


def test_matrix_reaches_every_instantiated_kernel():
    inst = cmx.instantiated()
    reached = {cmx.kernel_of(c) for c in cmx.CASES}
    assert None not in reached
    assert sorted(inst - reached) == [], "kernel paths no matrix case runs"
    assert sorted(reached - inst) == [], "the selection mirror names kernels vrgdg_inst.cuh does not build"


def test_every_kernel_runs_on_both_loaders_and_in_each_noise_mode():
    """each tile instantiation on the TMA and on the generic loader; grain chains in each noise mode on every dtype"""
    by_shape = {}
    for c in cmx.CASES:
        by_shape.setdefault(c.shape, set()).add(cmx.kernel_of(c))
    tiles = {k for k in cmx.instantiated() if k[0] == "tile"}
    assert tiles <= by_shape["tma"] | by_shape["groups"]
    assert tiles <= by_shape["ragged"] | by_shape["notma"]
    for dt in cmx.DTYPES:
        for nz in cmx.NOISES:
            assert any(c.grain and c.dtype == dt and c.noise == nz and c.stencil and c.post for c in cmx.CASES), (dt, nz)


def test_matrix_axes():
    ids = [cmx.case_id(c) for c in cmx.CASES]
    assert len(ids) == len(set(ids))
    assert {c.schedule for c in cmx.CASES if c.cm} == set(cmx.SCHEDULES)
    assert {c.stencil for c in cmx.CASES} == set(cmx.STENCIL_PAIRS) | {None}
    assert {c.dtype for c in cmx.CASES} == set(cmx.DTYPES)
    assert cmx.SHAPES["groups"][0] >= 5
    # the TMA shape spans several tiles in both directions and keeps rows 16-byte aligned for every dtype
    B, H, W = cmx.SHAPES["tma"]
    assert H > 2 * 32 and 3 * W > 2 * 240 and (3 * W) % 16 == 0 and W % 4 == 0
    assert cmx.SHAPES["ragged"][2] % 4 != 0


def test_kernel_mirror_spot_checks():
    C = cmx.Case
    # the benchmarked chain: in-kernel noise, f-planes, LUT, unsharp -> the inexact f-plane tile kernel
    assert cmx.kernel_of(C(1, 1, 1, 0, (1, 0), "f32", "clip", "g2", "groups")) == ("tile", "f32", cmx.ST_CMF | cmx.ST_LUT, False)
    # the same chain on external noise in exact arithmetic, and on the recompute schedule
    assert cmx.kernel_of(C(1, 1, 1, 0, (1, 0), "f32", "ext", "default", "tma")) == ("tile", "f32", cmx.ST_CMF | cmx.ST_LUT, True)
    assert cmx.kernel_of(C(1, 1, 1, 0, (1, 0), "f32", "ext", "recompute", "groups")) == ("tile", "f32", 7, True)
    # ragged fp32 frames cannot take the f-planes
    assert cmx.kernel_of(C(0, 1, 0, 0, (1, 0), "f32", "none", "default", "ragged")) == ("tile", "f32", cmx.ST_CM, True)
    # post grain alone runs through the grain plane; behind a pre-stage it does not
    assert cmx.kernel_of(C(0, 0, 0, 1, None, "u8", "none", "default", "tma")) == ("tile", "u8", cmx.ST_POST, True)
    assert cmx.kernel_of(C(0, 0, 1, 1, None, "u8", "none", "default", "tma")) == ("tile", "u8", cmx.ST_LUT, True)
    # 16-bit stencils never keep the NumPy evaluation order; in-kernel noise drops it on fp32 too
    assert not cmx.exact_stencil(C(0, 0, 0, 0, (1, 0), "f16", "none", "default", "tma"))
    assert not cmx.exact_stencil(C(1, 0, 0, 0, (1, 0), "f32", "frame", "default", "tma"))
    assert cmx.exact_stencil(C(1, 0, 1, 0, (4, 0), "u8", "ext", "default", "tma"))


def test_error_bars():
    C = cmx.Case
    assert cmx.float_bar(C(1, 0, 1, 0, (4, 0), "f32", "ext", "default", "tma")) == 0
    assert cmx.float_bar(C(1, 0, 1, 0, (1, 1), "f32", "ext", "default", "tma")) == 0
    assert cmx.float_bar(C(1, 0, 1, 0, (3, 1), "f32", "ext", "default", "tma")) == 1e-5
    assert cmx.float_bar(C(1, 0, 0, 0, None, "f32", "frame", "default", "tma")) == 4e-6
    assert cmx.float_bar(C(1, 1, 1, 1, (1, 0), "f32", "ext", "default", "tma")) == 1e-5 + 1e-6
    assert cmx.half_bar(C(0, 1, 0, 0, None, "bf16", "none", "default", "tma")) == 2.0 ** -8 + 1e-5

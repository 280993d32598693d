"""The kernels' per-pixel arithmetic header (csrc/vrgdg_math.cuh) compiled for the HOST (tests/hostcheck) against the
golden vectors: catches index / rounding mistakes on a machine without a GPU.  The GPU tests repeat the comparison on
the real kernels."""
import ctypes
import os

import numpy as np
import torch

from helpers import LUTS, load_golden, t

vp, i64, f32, ci = ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_int


def P(a):
    return a.ctypes.data_as(vp)


def flat(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32).reshape(-1, 3))


def test_philox4x32_10_known_answers(hostcheck):
    """Random123 kat_vectors for philox4x32-10."""
    cases = [([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
             ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
             ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0], [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1])]
    for ctr, key, want in cases:
        c, k, o = np.array(ctr, dtype=np.uint32), np.array(key, dtype=np.uint32), np.zeros(4, dtype=np.uint32)
        hostcheck.hc_philox(P(c), P(k), P(o))
        assert o.tolist() == want


def test_normals_are_standard_and_keyed(hostcheck):
    """generator definition: one Philox call per horizontal pixel pair, counter (x>>1, y, frame words)."""
    sig = [ctypes.c_uint64, i64, i64, ci, ci, ci, ci, vp]
    hostcheck.hc_normals.argtypes = sig
    hostcheck.hc_normals_pairs.argtypes = sig
    W, R = 640, 300
    a = np.zeros((R, W, 3), dtype=np.float32)
    hostcheck.hc_normals(42, 0, 0, 0, W, 0, R, P(a))
    assert abs(a.mean()) < 0.01 and abs(a.var() - 1.0) < 0.01 and abs((a.astype(np.float64) ** 4).mean() - 3.0) < 0.1
    assert np.abs(a).max() > 4.0 and np.abs(a).max() < 5.6           # 21-bit radius field: |z| <= 5.52
    for c0, c1 in ((0, 1), (0, 2), (1, 2)):
        assert abs((a[..., c0] * a[..., c1]).mean()) < 0.01
    assert abs((a[:, :-1, 0] * a[:, 1:, 0]).mean()) < 0.01 and abs((a[:, 0::2, 2] * a[:, 1::2, 0]).mean()) < 0.01   # within a pair too
    ap = np.zeros_like(a)
    hostcheck.hc_normals_pairs(42, 0, 0, 0, W, 0, R, P(ap))           # pair interface == per-pixel interface
    assert np.array_equal(a, ap)
    b = np.zeros_like(a)
    hostcheck.hc_normals(42, 5, 0, 0, W, 0, R, P(b))                  # other frame
    assert np.abs(a - b).mean() > 0.5
    c = np.zeros((10, W, 3), dtype=np.float32)
    hostcheck.hc_normals(42, 0, 0, 0, W, 100, 10, P(c))               # a window of the same frame: counter-based
    assert np.array_equal(c, a[100:110])
    # odd width: same (x, y) -> same value regardless of the frame width
    d = np.zeros((4, 33, 3), dtype=np.float32)
    hostcheck.hc_normals(42, 0, 0, 0, 33, 0, 4, P(d))
    assert np.array_equal(d, a[:4, :33])
    # PER_FRAME mode: (seed + frame0 + i) & 0x7fffffff is what matters -> (40,2,0) == (42,0,0) == (30,5,7)
    e, f, g = (np.zeros((4, 64, 3), dtype=np.float32) for _ in range(3))
    hostcheck.hc_normals(40, 2, 0, 1, 64, 0, 4, P(e))
    hostcheck.hc_normals(42, 0, 0, 1, 64, 0, 4, P(f))
    hostcheck.hc_normals(30, 5, 7, 1, 64, 0, 4, P(g))
    assert np.array_equal(e, f) and np.array_equal(f, g) and not np.array_equal(e, a[:4, :64])


def test_grain_blend_exact_is_bit_identical(hostcheck):
    hostcheck.hc_grain.argtypes = [vp, vp, vp, i64, f32, f32, f32, ci]
    g = load_golden("grain")
    for tag in ("a", "odd"):
        x, z = flat(g[f"x_{tag}"]), flat(g[f"z_{tag}"])
        o = np.zeros_like(x)
        hostcheck.hc_grain(P(x), P(z), P(o), x.shape[0], 0.5, 0.5, 1.0 - 0.5, 1)
        assert np.array_equal(o, flat(g[f"out_{tag}_i50_s50"]))
        hostcheck.hc_grain(P(x), P(z), P(o), x.shape[0], 0.04, 0.37, 1.0 - 0.37, 1)
        assert np.array_equal(o, flat(g[f"out_{tag}_i04_s37"]))
        hostcheck.hc_grain(P(x), P(z), P(o), x.shape[0], 0.04, 0.37, 1.0 - 0.37, 0)     # fused variant
        assert np.abs(o - flat(g[f"out_{tag}_i04_s37"])).max() < 1e-6


def test_lut_eval_exact_is_bit_identical(hostcheck, oracle):
    hostcheck.hc_lut3d.argtypes = [vp, vp, i64, vp, ci, vp, vp, f32, f32, ci]
    g = load_golden("lut")
    x = flat(g["x"])
    o = np.zeros_like(x)
    for fname in sorted(os.listdir(LUTS)):
        if not fname.endswith(".cube"):
            continue
        key = fname.split(".")[0].replace(" ", "_")
        d = oracle.parse_cube(os.path.join(LUTS, fname))
        lut = np.ascontiguousarray(d["lut"].numpy())
        dmin = d["domain_min"].numpy().copy()
        span = torch.clamp(d["domain_max"] - d["domain_min"], min=1e-6).numpy().copy()
        hostcheck.hc_lut3d(P(x), P(o), x.shape[0], P(lut), d["size"], P(dmin), P(span), 1.0, 0.0, 1)
        assert np.array_equal(o, flat(g[f"{key}__s10"])), fname
        blend = 3.5 / 10.0
        hostcheck.hc_lut3d(P(x), P(o), x.shape[0], P(lut), d["size"], P(dmin), P(span), blend, 1.0 - blend, 1)
        assert np.array_equal(o, flat(g[f"{key}__s3p5"])), fname
        hostcheck.hc_lut3d(P(x), P(o), x.shape[0], P(lut), d["size"], P(dmin), P(span), 1.0, 0.0, 0)      # contracted variant
        assert np.abs(o - flat(g[f"{key}__s10"])).max() < 1e-6
        hostcheck.hc_lut3d(P(x), P(o), x.shape[0], P(lut), d["size"], P(dmin), P(span), 1.0, 0.0, 2)      # two-pixel form
        assert np.array_equal(o, flat(g[f"{key}__s10"])), fname
        hostcheck.hc_lut3d(P(x), P(o), x.shape[0], P(lut), d["size"], P(dmin), P(span), blend, 1.0 - blend, 3)   # one channel per lane (tile kernels)
        assert np.array_equal(o, flat(g[f"{key}__s3p5"])), fname
        # polynomial cells of the fast chains (trilinear coefficients, 7 FMAs per channel): same cell and weights, values within
        # a few 1e-7 of the exact interpolation
        rng = max(1.0, float(lut.max() - lut.min()))
        hostcheck.hc_lut3d(P(x), P(o), x.shape[0], P(lut), d["size"], P(dmin), P(span), 1.0, 0.0, 4)
        assert np.abs(o - flat(g[f"{key}__s10"])).max() <= 5.0e-7 * rng, (fname, np.abs(o - flat(g[f"{key}__s10"])).max())
        hostcheck.hc_lut3d(P(x), P(o), x.shape[0], P(lut), d["size"], P(dmin), P(span), blend, 1.0 - blend, 4)
        assert np.abs(o - flat(g[f"{key}__s3p5"])).max() <= 5.0e-7 * rng, fname


def test_stencil_epilogues_and_colormatch_within_tolerance(hostcheck, oracle):
    hostcheck.hc_stencil.argtypes = [vp, vp, ci, ci, ci, f32, ci, ci]
    g = load_golden("stencil")
    x = np.ascontiguousarray(g["x"][0])
    o = np.zeros_like(x)
    for op, key, border in ((1, "unsharp_np", 0), (1, "unsharp_torch", 1), (2, "laplacian_np", 0), (3, "laplacian_torch", 1),
                            (4, "sobel_np", 0), (5, "sobel_torch", 1)):
        hostcheck.hc_stencil(P(x), P(o), x.shape[0], x.shape[1], op, 0.5, border, 0)
        assert np.abs(o - g[key][0]).max() <= 1e-5, key
    # exact epilogues: bit-identical to the NumPy paths (and to avg_pool2d for the zero-padded unsharp)
    for op, key, border, s in ((1, "unsharp_np", 0, 0.5), (2, "laplacian_np", 0, 0.5), (4, "sobel_np", 0, 0.5), (1, "unsharp_torch", 1, 0.5), (1, "unsharp_np_s10", 0, 10.0)):
        hostcheck.hc_stencil(P(x), P(o), x.shape[0], x.shape[1], op, s, border, 1)
        assert np.array_equal(o, g[key][0]), key
    xo = np.ascontiguousarray(g["x_odd"][0])
    oo = np.zeros_like(xo)
    for op, key in ((1, "unsharp_np_odd"), (2, "laplacian_np_odd"), (4, "sobel_np_odd")):
        hostcheck.hc_stencil(P(xo), P(oo), xo.shape[0], xo.shape[1], op, 1.3, 0, 1)
        assert np.array_equal(oo, g[key][0]), key
    hostcheck.hc_colormatch.argtypes = [vp, vp, i64, vp, f32, f32]
    c = load_golden("colormatch")
    ref_s = oracle.lab_moments_f64(t(c["ref"]))[0].numpy()
    for b in range(2):
        fs = oracle.lab_moments_f64(t(c["x"][b:b + 1]))[0].numpy()
        def stats(s):
            n, m = s[0], s[1:4] / s[0]
            var = (s[4:7] - s[1:4] * m) / (n - 1)
            return m.astype(np.float32), np.sqrt(var).astype(np.float32) + np.float32(1e-5)
        (mi, si), (mr, sr) = stats(fs), stats(ref_s)
        k = sr.astype(np.float64) / si.astype(np.float64)
        params = np.concatenate([k.astype(np.float32), (mr.astype(np.float64) - mi.astype(np.float64) * k).astype(np.float32), mi, si]).astype(np.float32)
        xin = flat(c["x"][b])
        out = np.zeros_like(xin)
        hostcheck.hc_colormatch(P(xin), P(out), xin.shape[0], P(params), 1.0, 0.0)
        assert np.abs(out - flat(c["out_t100"][b])).max() <= 1e-5
        hostcheck.hc_colormatch(P(xin), P(out), xin.shape[0], P(params), 0.6, 1.0 - 0.6)
        assert np.abs(out - flat(c["out_t60"][b])).max() <= 1e-5


def test_refined_powers_accuracy(hostcheck):
    """x^2.4, x^(1/3) of the colour match's input side: MUFU-style seed (perturbed by 3e-7 in the host build) + one division-free
    Newton step on the inverse root must land within a few fp32 roundings of the true power"""
    hostcheck.hc_pows.argtypes = [vp, vp, vp, vp, i64]
    x = np.exp(np.linspace(np.log(0.008856), np.log(2.0), 200001)).astype(np.float32)
    p24, pinv, cb = np.zeros_like(x), np.zeros_like(x), np.zeros_like(x)
    hostcheck.hc_pows(P(x), P(p24), P(pinv), P(cb), x.shape[0])
    x64 = x.astype(np.float64)
    assert np.abs(cb / np.cbrt(x64) - 1.0).max() < 4e-7
    assert np.abs(p24 / x64 ** 2.4 - 1.0).max() < 8e-7                       # (x * x^-0.2)^3: three times the error of the refined root
    assert np.abs(pinv / x64 ** (1.0 / 2.4) - 1.0).max() < 8e-7


def test_fspace_moments_equal_lab_moments(hostcheck, oracle):
    """the moments kernel sums (fy, fx-fy, fy-fz) and converts to Lab sums in fp64 (csrc/vrgdg_math.cuh::cm_sums_to_lab_host)"""
    hostcheck.hc_lab_sums.argtypes = [vp, i64, vp]
    c = load_golden("colormatch")
    for b in range(2):
        xin = flat(c["x"][b])
        got = np.zeros(7, dtype=np.float64)
        hostcheck.hc_lab_sums(P(xin), xin.shape[0], P(got))
        ref = oracle.lab_moments_f64(t(c["x"][b:b + 1]))[0].numpy()
        n = ref[0]
        assert got[0] == n
        assert np.abs(got[1:4] - ref[1:4]).max() / n < 5e-5
        assert np.allclose(got[4:7], ref[4:7], rtol=5e-6, atol=0.0)


def test_div_const_keeps_infinities(hostcheck):
    hostcheck.hc_div_const.argtypes = [vp, vp, i64, ci]
    x = np.array([np.inf, -np.inf, np.nan], dtype=np.float32)
    o = np.empty_like(x)
    for d in (9, 25, 49, 81, 255):
        hostcheck.hc_div_const(P(x), P(o), 3, d)
        assert o[0] == np.inf and o[1] == -np.inf and np.isnan(o[2])


def test_div_const_is_the_correctly_rounded_quotient(hostcheck):
    """div_const<D> (3 instructions: q = a*r, q' = fma(fma(-D, q, a), r, q)) against IEEE division on 8 M random finite bit patterns per
    divisor plus the special values; the GPU-side exhaustive run over all 2^32 patterns is tools/divconst_check.cu.
    The one representational difference: -0.0 -> +0.0."""
    hostcheck.hc_div_const.argtypes = [vp, vp, i64, ci]
    rng = np.random.default_rng(5)
    bits = rng.integers(0, 2 ** 32, size=8_000_000, dtype=np.uint64).astype(np.uint32)
    special = np.array([0x00000000, 0x00000001, 0x007FFFFF, 0x00800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x3F800000, 0x41100000, 0x80000001], dtype=np.uint32)
    x = np.concatenate([bits, special]).view(np.float32)
    x = x[np.isfinite(x)]                                                   # +-inf / NaN: test_div_const_keeps_infinities
    o = np.empty_like(x)
    with np.errstate(all="ignore"):
        for d in (9, 25, 49, 81, 255):
            hostcheck.hc_div_const(P(x), P(o), x.shape[0], d)
            ref = x / np.float32(d)
            assert np.array_equal(o.view(np.uint32), ref.view(np.uint32)), d
    z = np.array([-0.0], dtype=np.float32)
    hostcheck.hc_div_const(P(z), P(o), 1, 9)
    assert o[0] == 0.0                                                      # value equal; the sign of zero is not preserved


def test_coefficient_cells_random_tables_vs_float64_trilinear(hostcheck):
    """the fast chains' lookup (coefficient cells, 7 FMAs per channel; same code as the kernels, compiled for the host) on RANDOM tables of
    several sizes, value ranges and input domains against a float64 evaluation of the trilinear formula: the error stays within a few
    fp32 roundings of the table range whatever the table looks like (no smoothness assumed), and cell index / fractions are shared with
    the exact path (whose result is compared with the same float64 evaluation)"""
    hostcheck.hc_lut3d.argtypes = [vp, vp, i64, vp, ci, vp, vp, f32, f32, ci]
    rng = np.random.default_rng(20260924)
    for S, lo, hi in ((2, 0.0, 1.0), (9, -0.5, 1.5), (17, 0.0, 1.0), (33, -2.0, 3.0)):
        lut = rng.uniform(lo, hi, size=(S, S, S, 3)).astype(np.float32)
        dmin = np.array([0.05, 0.0, -0.1], dtype=np.float32)
        span = np.array([0.9, 1.0, 1.3], dtype=np.float32)
        x = rng.uniform(-0.2, 1.2, size=(20000, 3)).astype(np.float32)
        x[:64] = rng.integers(0, S, size=(64, 3)).astype(np.float32) / np.float32(S - 1) * span + dmin      # some points on the lattice
        # float64 trilinear on the float32 coordinates the kernels form (division, clamp, scale in fp32: the index math is shared)
        n = np.clip(((x - dmin) / span).astype(np.float32), np.float32(0), np.float32(1))
        c = (n * np.float32(S - 1)).astype(np.float32)
        i0 = np.floor(c).astype(np.int64)
        i1 = np.minimum(i0 + 1, S - 1)
        f = (c - i0.astype(np.float32)).astype(np.float64)
        L = lut.astype(np.float64)
        r0, g0, b0, r1, g1, b1 = i0[:, 0], i0[:, 1], i0[:, 2], i1[:, 0], i1[:, 1], i1[:, 2]
        fr, fg, fb = f[:, 0:1], f[:, 1:2], f[:, 2:3]
        c00 = L[b0, g0, r0] * (1 - fb) + L[b1, g0, r0] * fb
        c01 = L[b0, g1, r0] * (1 - fb) + L[b1, g1, r0] * fb
        c10 = L[b0, g0, r1] * (1 - fb) + L[b1, g0, r1] * fb
        c11 = L[b0, g1, r1] * (1 - fb) + L[b1, g1, r1] * fb
        want = np.clip((c00 * (1 - fg) + c01 * fg) * (1 - fr) + (c10 * (1 - fg) + c11 * fg) * fr, 0.0, 1.0)
        o = np.zeros_like(x)
        bound = 1.0e-6 * max(1.0, hi - lo)
        hostcheck.hc_lut3d(P(x), P(o), x.shape[0], P(lut), S, P(dmin), P(span), 1.0, 0.0, 1)          # exact path (corner cells)
        assert np.abs(o - want).max() <= bound, (S, "exact", np.abs(o - want).max())
        hostcheck.hc_lut3d(P(x), P(o), x.shape[0], P(lut), S, P(dmin), P(span), 1.0, 0.0, 4)          # coefficient cells
        assert np.abs(o - want).max() <= bound, (S, "coefficients", np.abs(o - want).max())

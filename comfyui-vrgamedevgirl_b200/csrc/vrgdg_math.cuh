// vrgdg_math.cuh — per-pixel arithmetic of the post-processing hot path.
//
// Everything here is __host__ __device__ so that tests/hostcheck can compile the very same
// arithmetic with g++ and compare it with the oracle on a machine without a GPU.  The product
// only ever runs the __device__ instantiation (the library has no CPU execution path).
//
// "x" suffix = exact: one IEEE fp32 rounding per operation, no FMA contraction, so results are
// bit-identical to the reference's CPU tensor ops (each of which rounds once).
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <math.h>

#if defined(__CUDACC__)
#define VRGDG_HD __host__ __device__ __forceinline__
#else
#define VRGDG_HD inline
#endif

namespace vrgdg {

// ---- exact fp32 primitives ---------------------------------------------------------------
#if defined(__CUDA_ARCH__)
VRGDG_HD float addx(float a, float b) { return __fadd_rn(a, b); }
VRGDG_HD float subx(float a, float b) { return __fsub_rn(a, b); }
VRGDG_HD float mulx(float a, float b) { return __fmul_rn(a, b); }
VRGDG_HD float divx(float a, float b) { return __fdiv_rn(a, b); }
VRGDG_HD float sqrtx(float a) { return __fsqrt_rn(a); }
#else
// host build uses -ffp-contract=off; volatile keeps the optimiser from re-associating
VRGDG_HD float addx(float a, float b) { volatile float r = a + b; return r; }
VRGDG_HD float subx(float a, float b) { volatile float r = a - b; return r; }
VRGDG_HD float mulx(float a, float b) { volatile float r = a * b; return r; }
VRGDG_HD float divx(float a, float b) { volatile float r = a / b; return r; }
VRGDG_HD float sqrtx(float a) { return sqrtf(a); }
#endif

VRGDG_HD float clamp01(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }

// a / D for the integer constants the exact kernels divide by (9, 25, 49, 81, 255): q = a*r, q' = fma(fma(-D, q, a), r, q) with
// r = RN(1/D) is the correctly rounded quotient for every FINITE fp32 a (all finite bit patterns, subnormals included, compared
// with __fdiv_rn on the GPU: tools/divconst_check.cu), 3 instructions instead of the ~9 of an IEEE division.  Outside that:
// a = -0.0 gives +0.0 (equal value); a = +-inf would give NaN (inf - inf in the residual), so a select returns q = a*r = +-inf
// there, as IEEE division does (synthetic / HDR inputs can hold inf; NaN stays NaN either way).
// Not valid for non-integer divisors (0.45 fails 0.7 % of inputs).
template <int D>
VRGDG_HD float div_const(float a) {
  static_assert(D == 9 || D == 25 || D == 49 || D == 81 || D == 255, "divisor not covered by the exhaustive check");
  const float r = 1.0f / (float)D;
#if defined(__CUDA_ARCH__)
  const float q = __fmul_rn(a, r);
  const float v = __fmaf_rn(__fmaf_rn(-(float)D, q, a), r, q);
  return (fabsf(a) == INFINITY) ? q : v;
#else
  const float q = mulx(a, r);
  const float v = fmaf(fmaf(-(float)D, q, a), r, q);
  return (fabsf(a) == INFINITY) ? q : v;
#endif
}

// ---- Philox4x32-10 (Salmon et al., SC'11), counter-based ----------------------------------
struct U4 { uint32_t x, y, z, w; };

VRGDG_HD void mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
#if defined(__CUDA_ARCH__)
  lo = a * b;
  hi = __umulhi(a, b);
#else
  uint64_t p = (uint64_t)a * (uint64_t)b;
  lo = (uint32_t)p;
  hi = (uint32_t)(p >> 32);
#endif
}

constexpr int PHILOX_ROUNDS = 10;
constexpr uint32_t PHILOX_W0 = 0x9E3779B9u, PHILOX_W1 = 0xBB67AE85u;

// Round keys are a function of the key only -> evaluated once on the host and read from the kernel's constant
// bank (no registers, no per-pixel key schedule).
struct GrainKey {
  uint32_t rk[PHILOX_ROUNDS][2];
};

VRGDG_HD U4 philox4x32_rk(U4 c, const GrainKey& K) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
#pragma unroll
  for (int r = 0; r < PHILOX_ROUNDS; ++r) {
    uint32_t h0, l0, h1, l1;
    mulhilo(M0, c.x, h0, l0);
    mulhilo(M1, c.z, h1, l1);
    U4 n;
    n.x = h1 ^ c.y ^ K.rk[r][0];
    n.y = l1;
    n.z = h0 ^ c.w ^ K.rk[r][1];
    n.w = l0;
    c = n;
  }
  return c;
}

// Grain generator (documented in DESIGN.md).  One Philox call serves a horizontal PIXEL PAIR (x>>1):
//   counter = (x >> 1, y, fw0, fw1), key -> round keys K
//   VRGDG_SEED_PER_CLIP : key = (seed_lo, seed_hi);            (fw0, fw1) = absolute frame index frame0+i
//   VRGDG_SEED_PER_FRAME: key = ("VRGD", "B200") constants;    (fw0, fw1) = ((seed+frame0+i) & 0x7FFFFFFF, 0xFFFFFFFF)
//                         (EnhancerNodes.py:267-268 seeds one generator per frame with exactly that value)
// The 128 output bits are cut into six 21-bit fields = three Box-Muller (radius, angle) pairs = six normals:
//   pixel 0 of the pair: z_r, z_g = pair A (cos, sin), z_b = pair B (cos);  pixel 1: z_r = pair B (sin), z_g, z_b = pair C.
inline void grain_make_key(uint64_t seed, int seed_mode, GrainKey& K) {
  uint32_t k0 = (seed_mode == 1) ? 0x56524744u : (uint32_t)seed;
  uint32_t k1 = (seed_mode == 1) ? 0x42323030u : (uint32_t)(seed >> 32);
  for (int r = 0; r < PHILOX_ROUNDS; ++r) {
    K.rk[r][0] = k0 + (uint32_t)r * PHILOX_W0;
    K.rk[r][1] = k1 + (uint32_t)r * PHILOX_W1;
  }
}

struct GrainFrame { uint32_t f0, f1; };

VRGDG_HD GrainFrame grain_frame(uint64_t seed, int64_t frame0, int64_t frame_in_batch, int seed_mode) {
  GrainFrame g;
  if (seed_mode == 1) {
    g.f0 = (uint32_t)((uint64_t)((int64_t)seed + frame0 + frame_in_batch) & 0x7FFFFFFFull);
    g.f1 = 0xFFFFFFFFu;
  } else {
    uint64_t f = (uint64_t)(frame0 + frame_in_batch);
    g.f0 = (uint32_t)f;
    g.f1 = (uint32_t)(f >> 32);
  }
  return g;
}

VRGDG_HD U4 grain_pair_bits(const GrainKey& K, const GrainFrame& f, uint32_t xpair, uint32_t y) {
  U4 c;
  c.x = xpair; c.y = y; c.z = f.f0; c.w = f.f1;
  return philox4x32_rk(c, K);
}

// Box-Muller on 21-bit fields: u = (k + 0.5) 2^-21 in (0,1), theta = 2 pi k 2^-21
VRGDG_HD void box_muller21(uint32_t rad, uint32_t ang, float& c, float& s) {
  const float S21 = 4.76837158203125e-07f;              // 2^-21
  const float H21 = 2.384185791015625e-07f;             // 2^-22
  const float TWO_PI_S21 = 2.9960562263390644e-06f;     // 2 pi 2^-21
  float u = fmaf((float)rad, S21, H21);
  float th = (float)ang * TWO_PI_S21;
#if defined(__CUDA_ARCH__)
  // -2 ln u = -2 ln2 log2 u : MUFU.LG2, MUFU.SQRT, MUFU.SIN, MUFU.COS
  float l2, rr, sn, cs;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l2) : "f"(u));
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(rr) : "f"(l2 * -1.3862943611198906f));
  asm("sin.approx.ftz.f32 %0, %1;" : "=f"(sn) : "f"(th));
  asm("cos.approx.ftz.f32 %0, %1;" : "=f"(cs) : "f"(th));
#else
  float rr = sqrtf(-2.0f * logf(u));
  float sn = sinf(th), cs = cosf(th);
#endif
  c = rr * cs;
  s = rr * sn;
}

VRGDG_HD void grain_fields(U4 r, uint32_t* rad, uint32_t* ang) {
  const uint32_t M = 0x1FFFFFu;
  rad[0] = r.x & M;
  ang[0] = ((r.x >> 21) | (r.y << 11)) & M;
  rad[1] = (r.y >> 10) & M;
  ang[1] = r.z & M;
  rad[2] = ((r.z >> 21) | (r.w << 11)) & M;
  ang[2] = (r.w >> 10) & M;
}

// all six normals of a pair: z[0..2] = pixel 0 (r,g,b), z[3..5] = pixel 1
VRGDG_HD void grain_pair_normals(U4 r, float* z) {
  uint32_t rad[3], ang[3];
  grain_fields(r, rad, ang);
  float c0, s0, c1, s1, c2, s2;
  box_muller21(rad[0], ang[0], c0, s0);
  box_muller21(rad[1], ang[1], c1, s1);
  box_muller21(rad[2], ang[2], c2, s2);
  z[0] = c0; z[1] = s0; z[2] = c1;
  z[3] = s1; z[4] = c2; z[5] = s2;
}

// the three normals of one pixel of the pair (lane = x & 1): two Box-Muller evaluations
VRGDG_HD void grain_lane_normals(U4 r, int lane, float& zr, float& zg, float& zb) {
  uint32_t rad[3], ang[3];
  grain_fields(r, rad, ang);
  float c1, s1, ca, sa;
  box_muller21(rad[1], ang[1], c1, s1);
  box_muller21(lane ? rad[2] : rad[0], lane ? ang[2] : ang[0], ca, sa);
  zr = lane ? s1 : ca;
  zg = lane ? ca : sa;
  zb = lane ? sa : c1;
}

VRGDG_HD void grain_pixel_normals(const GrainKey& K, const GrainFrame& f, uint32_t x, uint32_t y, float& zr, float& zg, float& zb) {
  grain_lane_normals(grain_pair_bits(K, f, x >> 1, y), (int)(x & 1u), zr, zg, zb);
}

// ---- grain blend: nodes.py:53-60 ------------------------------------------------------------
// exact variant = the reference's op sequence, one rounding per op.
VRGDG_HD void grain_blend_exact(float& r, float& g, float& b, float zr, float zg, float zb,
                                float I, float s, float oms) {
  float zr2 = mulx(zr, 2.0f);                     // grain[...,0] *= 2.0
  float zb3 = mulx(zb, 3.0f);                     // grain[...,2] *= 3.0
  float gy = mulx(oms, zg);                       // (1.0 - s) * gray
  float gr = addx(mulx(s, zr2), gy);              // s*grain + (1-s)*gray
  float gg = addx(mulx(s, zg), gy);
  float gb = addx(mulx(s, zb3), gy);
  r = clamp01(addx(r, mulx(gr, I)));              // batch + grain*I ; clamp
  g = clamp01(addx(g, mulx(gg, I)));
  b = clamp01(addx(b, mulx(gb, I)));
}

// fused variant for in-kernel noise (the noise stream itself is ours, so contraction is free)
VRGDG_HD void grain_blend_fast(float& r, float& g, float& b, float zr, float zg, float zb,
                               float I, float s, float oms) {
  float gy = oms * zg;
  r = clamp01(fmaf(I, fmaf(2.0f * s, zr, gy), r));
  g = clamp01(fmaf(I, fmaf(s, zg, gy), g));
  b = clamp01(fmaf(I, fmaf(3.0f * s, zb, gy), b));
}

// ---- 3D LUT trilinear: VRGDG_IV_Adjustments.py:293-336 ------------------------------------------
// Device table layout ("cell table", built by lut_pack_entry / vrgdg_lut3d_pack): one 96-byte entry per cell origin
//   entry (b,g,r) = rgb x { c000 c100 c010 c110 c001 c101 c011 c111 },  cXYZ = lut[min(b+Z,S-1), min(g+Y,S-1), min(r+X,S-1), :]
// (channel-planar: one 32-byte sector per output channel) so a pixel fetches its 8 corners (24 floats) from THREE sectors at
// consecutive addresses (lut_load8) instead of 24 scalar loads - or three lanes fetch one sector each.  The gather is bound by L1 tag
// lookups per divergent lane, not by bytes: 3 sectors per pixel beat both a 32-byte r-pair table (4 per pixel) and scalar loads.
struct LutParams {
  const float* lut;      // cell table, S*S*S*24 floats: per cell three 32-byte sectors (R, G, B), 8 corners each
  const float* lutp;     // polynomial cell table (fast arithmetic only, see lutp_* below), same shape as `lut`
  int S;
  float smax;            // float(S-1)
  float dmin[3], dspan[3];
  float blend, one_minus_blend;
  int unit_domain;       // dmin == 0 and dspan == 1: (x-0)/1 == x exactly, the division is skipped
};

constexpr int LUT_CELL_FLOATS = 24;

struct F8 { float v[8]; };

// One 32-byte sector as two 128-bit non-coherent loads (LDG.E.128.CONSTANT): sm_90 has no 256-bit load, and both halves hit
// the same sector, so the L2 -> L1 traffic per corner set is unchanged.
VRGDG_HD F8 lut_load8(const float* p) {
  F8 q;
#if defined(__CUDA_ARCH__)
  asm("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];"
      : "=f"(q.v[0]), "=f"(q.v[1]), "=f"(q.v[2]), "=f"(q.v[3]) : "l"(p));
  asm("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+16];"
      : "=f"(q.v[4]), "=f"(q.v[5]), "=f"(q.v[6]), "=f"(q.v[7]) : "l"(p));
#else
  for (int i = 0; i < 8; ++i) q.v[i] = p[i];
#endif
  return q;
}

// one cell-table entry from the reference-layout table [S][S][S][3]
VRGDG_HD void lut_pack_entry(const float* lut3, int S, int b, int g, int r, float* dst24) {
  const int b1 = (b + 1 < S) ? b + 1 : S - 1, g1 = (g + 1 < S) ? g + 1 : S - 1, r1 = (r + 1 < S) ? r + 1 : S - 1;
  const int cb[8] = {b, b, b, b, b1, b1, b1, b1};
  const int cg[8] = {g, g, g1, g1, g, g, g1, g1};
  const int cr[8] = {r, r1, r, r1, r, r1, r, r1};
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float* a = lut3 + ((size_t)(cb[k] * S + cg[k]) * S + cr[k]) * 3;
    dst24[k] = a[0]; dst24[8 + k] = a[1]; dst24[16 + k] = a[2];     // channel-planar: one 32-byte sector per output channel
  }
}

// coordinate -> (cell index, fraction); bit-exact with :296-316
VRGDG_HD void lut_coord(float v, float dmin, float dspan, bool unit, float smax, int S, int& i0, int& i1, float& f) {
  float n = unit ? v : divx(subx(v, dmin), dspan);   // (source - domain_min) / domain_span
  n = clamp01(n);                                 // torch.clamp(normalized, 0, 1)
  float c = mulx(n, smax);                        // normalized * max_index
  float fl = floorf(c);
  i0 = (int)fl;                                   // torch.floor(r).long()
  i1 = (i0 + 1 < S - 1) ? i0 + 1 : S - 1;         // clamp(r0+1, max=max_index)
  f = subx(c, fl);                                // r - r0.float()
}

template <bool EXACT>
VRGDG_HD float lerp_ref(float a, float b, float f, float omf) {
  if (EXACT) return addx(mulx(a, omf), mulx(b, f));   // a*(1-f) + b*f, three roundings (:327-335)
  return fmaf(f, b - a, a);                           // contracted form for fused chains (<= 2e-7 away)
}

// one channel from its sector q = {c000 c100 c010 c110 c001 c101 c011 c111} (cXYZ: X = r, Y = g, Z = b neighbour), :318-339
template <bool EXACT>
VRGDG_HD float lut_channel(const F8& q, float fr, float fg, float fb, float omr, float omg, float omb) {
  const float c00 = lerp_ref<EXACT>(q.v[0], q.v[4], fb, omb);     // c000*(1-fb) + c001*fb
  const float c01 = lerp_ref<EXACT>(q.v[2], q.v[6], fb, omb);     // c010, c011
  const float c10 = lerp_ref<EXACT>(q.v[1], q.v[5], fb, omb);     // c100, c101
  const float c11 = lerp_ref<EXACT>(q.v[3], q.v[7], fb, omb);     // c110, c111
  const float c0 = lerp_ref<EXACT>(c00, c01, fg, omg);
  const float c1 = lerp_ref<EXACT>(c10, c11, fg, omg);
  return clamp01(lerp_ref<EXACT>(c0, c1, fr, omr));
}

template <bool EXACT>
VRGDG_HD void lut3d_eval(const LutParams& P, float& r, float& g, float& b) {
  int r0, r1, g0, g1, b0, b1;
  float fr, fg, fb;
  lut_coord(r, P.dmin[0], P.dspan[0], P.unit_domain != 0, P.smax, P.S, r0, r1, fr);
  lut_coord(g, P.dmin[1], P.dspan[1], P.unit_domain != 0, P.smax, P.S, g0, g1, fg);
  lut_coord(b, P.dmin[2], P.dspan[2], P.unit_domain != 0, P.smax, P.S, b0, b1, fb);
  (void)r1; (void)g1; (void)b1;                     // the clamped neighbours are baked into the cell entry
  const float* p = P.lut + (size_t)((b0 * P.S + g0) * P.S + r0) * LUT_CELL_FLOATS;
  const F8 q0 = lut_load8(p), q1 = lut_load8(p + 8), q2 = lut_load8(p + 16);
  const float omb = subx(1.0f, fb), omg = subx(1.0f, fg), omr = subx(1.0f, fr);
  r = lut_channel<EXACT>(q0, fr, fg, fb, omr, omg, omb);
  g = lut_channel<EXACT>(q1, fr, fg, fb, omr, omg, omb);
  b = lut_channel<EXACT>(q2, fr, fg, fb, omr, omg, omb);
}

// One output channel only: the element-mapped gather of the tile kernels (three lanes of a pixel read the three sectors of
// one cell, i.e. one or two 128-byte lines per PIXEL instead of three per pixel: the L1 data pipe counts wavefronts per
// distinct line and instruction; tools/lut_bench.cu compares the two mappings as v10 and v13).
template <bool EXACT>
VRGDG_HD float lut3d_eval_channel(const LutParams& P, float r, float g, float b, int ch) {
  int r0, r1, g0, g1, b0, b1;
  float fr, fg, fb;
  lut_coord(r, P.dmin[0], P.dspan[0], P.unit_domain != 0, P.smax, P.S, r0, r1, fr);
  lut_coord(g, P.dmin[1], P.dspan[1], P.unit_domain != 0, P.smax, P.S, g0, g1, fg);
  lut_coord(b, P.dmin[2], P.dspan[2], P.unit_domain != 0, P.smax, P.S, b0, b1, fb);
  (void)r1; (void)g1; (void)b1;
  const F8 q = lut_load8(P.lut + (size_t)((b0 * P.S + g0) * P.S + r0) * LUT_CELL_FLOATS + 8 * ch);
  return lut_channel<EXACT>(q, fr, fg, fb, subx(1.0f, fr), subx(1.0f, fg), subx(1.0f, fb));
}

// Two pixels at once: both address computations first, then all six sector loads, then the lerps, so that the two
// gathers overlap (the tile pre-stage is latency-bound on these loads).
struct LutCell { const float* p; float fr, fg, fb; };

VRGDG_HD LutCell lut_locate(const LutParams& P, float r, float g, float b) {
  int r0, r1, g0, g1, b0, b1;
  LutCell c;
  lut_coord(r, P.dmin[0], P.dspan[0], P.unit_domain != 0, P.smax, P.S, r0, r1, c.fr);
  lut_coord(g, P.dmin[1], P.dspan[1], P.unit_domain != 0, P.smax, P.S, g0, g1, c.fg);
  lut_coord(b, P.dmin[2], P.dspan[2], P.unit_domain != 0, P.smax, P.S, b0, b1, c.fb);
  (void)r1; (void)g1; (void)b1;
  c.p = P.lut + (size_t)((b0 * P.S + g0) * P.S + r0) * LUT_CELL_FLOATS;
  return c;
}

template <bool EXACT>
VRGDG_HD void lut_finish(const LutCell& c, const F8& q0, const F8& q1, const F8& q2, float& r, float& g, float& b) {
  const float omb = subx(1.0f, c.fb), omg = subx(1.0f, c.fg), omr = subx(1.0f, c.fr);
  r = lut_channel<EXACT>(q0, c.fr, c.fg, c.fb, omr, omg, omb);
  g = lut_channel<EXACT>(q1, c.fr, c.fg, c.fb, omr, omg, omb);
  b = lut_channel<EXACT>(q2, c.fr, c.fg, c.fb, omr, omg, omb);
}

template <bool EXACT>
VRGDG_HD void lut3d_eval2(const LutParams& P, float* a, float* b) {
  const LutCell ca = lut_locate(P, a[0], a[1], a[2]), cb = lut_locate(P, b[0], b[1], b[2]);
  const F8 a0 = lut_load8(ca.p), a1 = lut_load8(ca.p + 8), a2 = lut_load8(ca.p + 16);
  const F8 b0 = lut_load8(cb.p), b1 = lut_load8(cb.p + 8), b2 = lut_load8(cb.p + 16);
  lut_finish<EXACT>(ca, a0, a1, a2, a[0], a[1], a[2]);
  lut_finish<EXACT>(cb, b0, b1, b2, b[0], b[1], b[2]);
}

// ---- polynomial cells (fast arithmetic only) ----------------------------------------------------------
// The chains that draw their own grain run contracted arithmetic anyway (tolerance 1e-5), so their lookup reads a second table
// that holds, per cell and channel, the COEFFICIENTS of the trilinear polynomial instead of its corner values:
//   v(fr, fg, fb) = sum over X,Y,Z in {0,1} of k_XYZ fr^X fg^Y fb^Z,
//   k_000 = c000, k_100 = c100 - c000, k_010 = c010 - c000, k_110 = c110 - c100 - c010 + c000, ...  (differences along r, g, b)
// evaluated as a nested Horner form with 7 FMAs per channel (the corner form needs 7 lerps = 14 instructions):
//   v = (k000 + fb k001 + fg (k010 + fb k011)) + fr (k100 + fb k101 + fg (k110 + fb k111)).
// Same 96-byte channel-planar cell, coefficient k_XYZ in the slot of corner cXYZ; three sector loads per pixel as before.
// The coefficients are formed in double from the fp32 corners and rounded once; cell index and fractions are the exact path's.
// Difference to the exact interpolation: a few 1e-8 of the table values (rounding of coefficients and FMAs).
VRGDG_HD void lutp_pack_entry(const float* lut3, int S, int b, int g, int r, float* dst24) {
  float c[LUT_CELL_FLOATS];
  lut_pack_entry(lut3, S, b, g, r, c);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    double k[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) k[i] = (double)c[8 * ch + i];
#pragma unroll
    for (int bit = 1; bit < 8; bit <<= 1) {          // Moebius transform: slot i (bit set) -= slot i without that bit
#pragma unroll
      for (int i = 0; i < 8; ++i) if (i & bit) k[i] -= k[i ^ bit];
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) dst24[8 * ch + i] = (float)k[i];
  }
}

// one channel from its coefficient sector q (slot XYZ: X = r, Y = g, Z = b exponent; slot index = X + 2 Y + 4 Z)
VRGDG_HD float lutp_channel(const F8& q, float fr, float fg, float fb) {
  const float a0 = fmaf(fb, q.v[4], q.v[0]), b0 = fmaf(fb, q.v[5], q.v[1]);
  const float a1 = fmaf(fb, q.v[6], q.v[2]), b1 = fmaf(fb, q.v[7], q.v[3]);
  return clamp01(fmaf(fr, fmaf(fg, b1, b0), fmaf(fg, a1, a0)));
}

VRGDG_HD LutCell lutp_locate(const LutParams& P, float r, float g, float b) {
  LutCell c = lut_locate(P, r, g, b);
  c.p = P.lutp + (c.p - P.lut);
  return c;
}
VRGDG_HD void lutp_eval(const LutParams& P, float& r, float& g, float& b) {
  const LutCell c = lutp_locate(P, r, g, b);
  const F8 q0 = lut_load8(c.p), q1 = lut_load8(c.p + 8), q2 = lut_load8(c.p + 16);
  r = lutp_channel(q0, c.fr, c.fg, c.fb); g = lutp_channel(q1, c.fr, c.fg, c.fb); b = lutp_channel(q2, c.fr, c.fg, c.fb);
}
VRGDG_HD void lutp_eval2(const LutParams& P, float* a, float* b) {
  const LutCell ca = lutp_locate(P, a[0], a[1], a[2]), cb = lutp_locate(P, b[0], b[1], b[2]);
  const F8 a0 = lut_load8(ca.p), a1 = lut_load8(ca.p + 8), a2 = lut_load8(ca.p + 16);
  const F8 b0 = lut_load8(cb.p), b1 = lut_load8(cb.p + 8), b2 = lut_load8(cb.p + 16);
  a[0] = lutp_channel(a0, ca.fr, ca.fg, ca.fb); a[1] = lutp_channel(a1, ca.fr, ca.fg, ca.fb); a[2] = lutp_channel(a2, ca.fr, ca.fg, ca.fb);
  b[0] = lutp_channel(b0, cb.fr, cb.fg, cb.fb); b[1] = lutp_channel(b1, cb.fr, cb.fg, cb.fb); b[2] = lutp_channel(b2, cb.fr, cb.fg, cb.fb);
}

// strength blend of apply_lut (:355-359) on already-rounded LUT output `y` and input `x`
template <bool EXACT>
VRGDG_HD float lut_blend(float x, float y, float blend, float omb) {
  if (EXACT) return addx(mulx(x, omb), mulx(y, blend));
  return fmaf(y, blend, x * omb);
}

// ---- sRGB <-> CIE Lab (kornia.color restatement; formulas in SURVEY.md §8c) ------------------------
// Colour match runs in "f-space": Lab is an affine image of (fx, fy, fz) = lab_f(XYZ / white),
//   L = 116 fy - 16,  a = 500 (fx - fy),  b = 200 (fy - fz),
// so the kernels never form L, a, b: the moments pass accumulates fy, fx - fy, fy - fz (cm_sums_to_lab turns their raw sums
// into Lab sums in fp64), and the per-frame affine map  lab' = t (lab k + c0) + (1 - t) lab  is folded into three FMAs on
// the f values (cm_fold).  Algebraically identical to nodes.py:105-115; the roundings differ at the 1e-7 level (the colour
// match is tolerance-based: 1e-5 on RGB, kornia itself is unpinned).
// Fractional powers: the INPUT side (x^2.4, x^(1/3)) is a MUFU seed 2^(e*log2 x) (~1e-6 relative) plus ONE Newton step of the
// matching integer root (its error is amplified by sd_ref/sd_img and by the a/b differencing); the OUTPUT side x^(1/2.4) is the
// MUFU seed alone (error <= ~5e-7 on a [0,1] value, not amplified).
VRGDG_HD float approx_pow(float x, float e) {        // x > 0, relative error ~1e-6
#if defined(__CUDA_ARCH__)
  float l, r;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(l * e));
  return r;
#else
  return exp2f(log2f(x) * e) * (1.0f + 3e-7f);       // host build (tests only): perturbed so that the Newton step is exercised
#endif
}
VRGDG_HD float approx_rcp(float x) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
#else
  return 1.0f / x;
#endif
}
// The Newton steps run on the INVERSE roots (r = x^(-1/n)): r' = r (1 + 1/n - (x/n) r^n) needs no division, so a refined power
// costs two XU operations (lg2, ex2) instead of three (the statistics pass ran the XU pipe at 81 % with the reciprocal form).
// x^(1/3) = x r'^2 with r = x^(-1/3), x in (0, ~2]
VRGDG_HD float cbrt_pos(float x) {
  const float r = approx_pow(x, -0.33333334f);
  const float r3 = (r * r) * r;
  const float rn = r * fmaf(x * r3, -0.33333334f, 1.3333334f);       // r (4/3 - x r^3 / 3)
  return (x * rn) * rn;
}
// x^(-0.2), refined
VRGDG_HD float inv_root5_pos(float x) {
  const float r = approx_pow(x, -0.2f);
  const float r2 = r * r, r4 = r2 * r2;
  return r * fmaf((x * r) * r4, -0.2f, 1.2f);                        // r (6/5 - x r^5 / 5)
}
// x^0.2 = x (x^(-0.2))^4   (accuracy tests)
VRGDG_HD float root5_pos(float x) {
  const float r = inv_root5_pos(x);
  const float r2 = r * r;
  return x * (r2 * r2);
}
// x^2.4 = (x * x^(-0.2))^3
VRGDG_HD float pow_2p4(float x) {
  const float s = x * inv_root5_pos(x);
  return (s * s) * s;
}
// x^(1/2.4), refined: (x^(1/12))^5 with one Newton step on the 12th root (kept for the accuracy tests; the kernels use the seed)
VRGDG_HD float pow_inv2p4(float x) {
  float y = approx_pow(x, 0.083333336f);
  float y2 = y * y, y4 = y2 * y2, y8 = y4 * y4, y11 = (y8 * y2) * y;
  y = fmaf(fmaf(-y11, y, x), approx_rcp(12.0f * y11), y);    // y - (y^12 - x) / (12 y^11)
  y2 = y * y;
  return (y2 * y2) * y;
}

// Divisions by constants are multiplications by the rounded reciprocal (<= 1 ulp from the divided value).
// Both sides of each where() are evaluated (the power on an argument clamped into its own domain) and the result is SELECTED:
// written as a ternary around the power the compiler emits a divergent branch per channel (BSSY / BRA / BSYNC: 4 extra
// instructions per conditional and two passes for every warp that holds one dark pixel).
VRGDG_HD float srgb_to_linear(float c) {
  // where(c > 0.04045, ((c + 0.055) / 1.055) ** 2.4, c / 12.92)
  const float p = pow_2p4(fmaf(fmaxf(c, 0.04045f), (float)(1.0 / 1.055), (float)(0.055 / 1.055)));
  const float l = c * (float)(1.0 / 12.92);
  return (c > 0.04045f) ? p : l;
}
VRGDG_HD float linear_to_srgb(float l) {
  // where(l > 0.0031308, 1.055 * clamp(l, min=thr) ** (1/2.4) - 0.055, 12.92 * l)
  const float p = fmaf(1.055f, approx_pow(fmaxf(l, 0.0031308f), 0.41666666f), -0.055f);
  const float q = 12.92f * l;
  return (l > 0.0031308f) ? p : q;
}
VRGDG_HD float lab_f(float t) {
  // where(t > 0.008856, clamp(t, min=0.008856) ** (1/3), 7.787 t + 4/29)
  const float p = cbrt_pos(fmaxf(t, 0.008856f));
  const float q = fmaf(7.787f, t, (float)(4.0 / 29.0));
  return (t > 0.008856f) ? p : q;
}
// rgb -> (fx, fy, fz): sRGB decode, OpenCV D65 matrix with the white point (0.95047, 1, 1.08883) folded into its rows, lab_f
VRGDG_HD void rgb_to_fxyz(float r, float g, float b, float& fx, float& fy, float& fz) {
  const float lr = srgb_to_linear(r), lg = srgb_to_linear(g), lb = srgb_to_linear(b);
  const float x = fmaf((float)(0.180423 / 0.95047), lb, fmaf((float)(0.357580 / 0.95047), lg, (float)(0.412453 / 0.95047) * lr));
  const float y = fmaf(0.072169f, lb, fmaf(0.715160f, lg, 0.212671f * lr));
  const float z = fmaf((float)(0.950227 / 1.08883), lb, fmaf((float)(0.119193 / 1.08883), lg, (float)(0.019334 / 1.08883) * lr));
  fx = lab_f(x); fy = lab_f(y); fz = lab_f(z);
}
VRGDG_HD void rgb_to_lab(float r, float g, float b, float& L, float& A, float& Bv) {
  float fx, fy, fz;
  rgb_to_fxyz(r, g, b, fx, fy, fz);
  L = fmaf(116.0f, fy, -16.0f);
  A = 500.0f * (fx - fy);
  Bv = 200.0f * (fy - fz);
}
VRGDG_HD float lab_finv(float f) {
  // where(f > 0.2068966, f ** 3, (f - 4/29) / 7.787)
  return (f > 0.2068966f) ? (f * f) * f : (f - (float)(4.0 / 29.0)) * (float)(1.0 / 7.787);
}
// (fx, fy, fz) -> rgb, clipped (kornia lab_to_rgb(clip=True) followed by nodes.py:121 clamp); fz >= 0 is the caller's job
VRGDG_HD void fxyz_to_rgb(float fx, float fy, float fz, float& r, float& g, float& b) {
  const float x = lab_finv(fx), y = lab_finv(fy), z = lab_finv(fz);       // XYZ / white; the white point is folded into the columns below
  const float lr = fmaf((float)(-0.4985363261688878 * 1.08883), z, fmaf(-1.5371515162713185f, y, (float)(3.2404813432005266 * 0.95047) * x));
  const float lg = fmaf((float)(0.0415559265582928 * 1.08883), z, fmaf(1.8759900014898907f, y, (float)(-0.9692549499965682 * 0.95047) * x));
  const float lb = fmaf((float)(1.0573110696453443 * 1.08883), z, fmaf(-0.2040413383665112f, y, (float)(0.0556466391351772 * 0.95047) * x));
  r = clamp01(linear_to_srgb(lr));
  g = clamp01(linear_to_srgb(lg));
  b = clamp01(linear_to_srgb(lb));
}
VRGDG_HD void lab_to_rgb(float L, float A, float Bv, float& r, float& g, float& b) {
  const float fy = (L + 16.0f) * (float)(1.0 / 116.0);
  fxyz_to_rgb(fmaf(A, (float)(1.0 / 500.0), fy), fy, fmaxf(fmaf(Bv, (float)(-1.0 / 200.0), fy), 0.0f), r, g, b);
}

// nodes.py:112-115: matched = (lab - mu)/sd * sd_ref + mu_ref ; blended = t*matched + (1-t)*lab
// p = {k[3] = sd_ref/sd_img, c0[3] = mu_ref - mu_img*k, mu_img[3], sd_img[3]}  (k and c0 are formed once per frame in fp64), so
// matched = lab*k + c0 and blended = lab*(t*k + (1-t)) + t*c0.  In f-space:
//   fy' = (L' + 16)/116 = fy*K_L + (t*c0_L - 16 K_L + 16)/116
//   fx' = a'/500 + fy'  = (fx - fy)*K_a + t*c0_a/500 + fy'
//   fz' = fy' - b'/200  = fy' - (fy - fz)*K_b - t*c0_b/200        (then max(fz', 0) as kornia does)
struct CmFold { float ky, cy, ka, ca, kb, cb; };
VRGDG_HD CmFold cm_fold(const float* p, float t, float omt) {
  CmFold f;
  f.ky = fmaf(t, p[0], omt);
  f.ka = fmaf(t, p[1], omt);
  f.kb = fmaf(t, p[2], omt);
  f.cy = fmaf(-16.0f, f.ky, fmaf(t, p[3], 16.0f)) * (float)(1.0 / 116.0);
  f.ca = (t * p[4]) * (float)(1.0 / 500.0);
  f.cb = (t * p[5]) * (float)(1.0 / 200.0);
  return f;
}
VRGDG_HD void colormatch_fold_pixel(float& r, float& g, float& b, const CmFold& f) {
  float fx, fy, fz;
  rgb_to_fxyz(r, g, b, fx, fy, fz);
  const float fy2 = fmaf(fy, f.ky, f.cy);
  const float fx2 = fmaf(fx - fy, f.ka, fy2 + f.ca);
  const float fz2 = fmaxf(fmaf(fz - fy, f.kb, fy2 - f.cb), 0.0f);
  fxyz_to_rgb(fx2, fy2, fz2, r, g, b);
}
// the same map applied to stored (fx, fy, fz): the second pass of the f-plane schedule
VRGDG_HD void colormatch_from_f(float& r, float& g, float& b, const CmFold& f) {
  const float fx = r, fy = g, fz = b;
  const float fy2 = fmaf(fy, f.ky, f.cy);
  const float fx2 = fmaf(fx - fy, f.ka, fy2 + f.ca);
  const float fz2 = fmaxf(fmaf(fz - fy, f.kb, fy2 - f.cb), 0.0f);
  fxyz_to_rgb(fx2, fy2, fz2, r, g, b);
}
VRGDG_HD void colormatch_pixel(float& r, float& g, float& b, const float* p, float t, float omt) {
  colormatch_fold_pixel(r, g, b, cm_fold(p, t, omt));
}

// Raw sums of the moments pass are over u = (fy, fx - fy, fy - fz): {n, S_u[3], S_uu[3]}.  Lab = (116 u0 - 16, 500 u1, 200 u2):
//   S_L = 116 S_0 - 16 n ;  S_LL = 116^2 S_00 - 2*116*16 S_0 + 256 n ;  S_a = 500 S_1 ; S_aa = 500^2 S_11 ; S_b = 200 S_2 ; S_bb = 200^2 S_22
inline void cm_sums_to_lab_host(const double* u, double* lab) {   // documentation of the fp64 fold in k_moments_final
  lab[0] = u[0];
  lab[1] = 116.0 * u[1] - 16.0 * u[0];
  lab[2] = 500.0 * u[2];
  lab[3] = 200.0 * u[3];
  lab[4] = 13456.0 * u[4] - 3712.0 * u[1] + 256.0 * u[0];
  lab[5] = 250000.0 * u[5];
  lab[6] = 40000.0 * u[6];
}

// ---- 3x3 stencil epilogues: nodes.py:194-207, :278-287, :369-382 (numpy) and :171-174,:249-258,:345-349 (torch)
// n[0..8] = row-major 3x3 neighbourhood, n[4] = centre.
VRGDG_HD float stencil_epilogue(int op, const float* n, float s) {
  float c = n[4], v;
  switch (op) {
    case 1: {  // box unsharp: blur = sum9 / 9 ; out = c + s*(c - blur)
      float sum = ((n[0] + n[1]) + n[2]) + ((n[3] + n[4]) + n[5]) + ((n[6] + n[7]) + n[8]);
      float blur = sum / 9.0f;
      v = c + s * (c - blur);
    } break;
    case 2: {  // numpy laplacian: lap = W + N + S + E - 4c ; out = c + s*lap   (blurs; reference quirk D5)
      float lap = (((n[3] + n[1]) + n[7]) + n[5]) - 4.0f * c;
      v = c + s * lap;
    } break;
    case 3: {  // torch laplacian: edges = 4c - N - S - E - W
      float e = 4.0f * c - n[1] - n[3] - n[5] - n[7];
      v = c + s * e;
    } break;
    case 4:
    case 5: {  // sobel
      float gx = (-n[0] - 2.0f * n[3] - n[6]) + (n[2] + 2.0f * n[5] + n[8]);
      float gy = (-n[0] - 2.0f * n[1] - n[2]) + (n[6] + 2.0f * n[7] + n[8]);
      float m = gx * gx + gy * gy + ((op == 5) ? 1e-6f : 0.0f);
      v = c + s * sqrtf(m);
    } break;
    default: v = c;
  }
  return clamp01(v);
}

// Exact variants: the NumPy path's evaluation order with one rounding per operation -> bit-identical to the
// reference's CPU sharpen nodes for fp32 frames (nodes.py:194-207, :278-287, :369-382).  The torch paths' convolutions
// (F.conv2d) have no defined summation order; for them (ops 3 and 5) this falls back to the fast epilogue.
VRGDG_HD float stencil_epilogue_exact(int op, const float* n, float s) {
  const float c = n[4];
  float v;
  switch (op) {
    case 1: {   // blur = (p00+p01+p02+p10+p11+p12+p20+p21+p22)/9.0, left to right ; out = img + s*(img - blur)
      float sum = addx(addx(addx(addx(addx(addx(addx(addx(n[0], n[1]), n[2]), n[3]), n[4]), n[5]), n[6]), n[7]), n[8]);
      float blur = div_const<9>(sum);                 // == sum / 9.0 (see div_const)
      v = addx(c, mulx(s, subx(c, blur)));
    } break;
    case 2: {   // lap = W + N + S + E - 4.0*img ; out = img + s*lap
      float lap = subx(addx(addx(addx(n[3], n[1]), n[7]), n[5]), mulx(4.0f, c));
      v = addx(c, mulx(s, lap));
    } break;
    case 4: {   // gx = -p00 - 2*p10 - p20 + p02 + 2*p12 + p22 ; gy = -p00 - 2*p01 - p02 + p20 + 2*p21 + p22
      float gx = addx(addx(addx(subx(subx(-n[0], mulx(2.0f, n[3])), n[6]), n[2]), mulx(2.0f, n[5])), n[8]);
      float gy = addx(addx(addx(subx(subx(-n[0], mulx(2.0f, n[1])), n[2]), n[6]), mulx(2.0f, n[7])), n[8]);
      v = addx(c, mulx(s, sqrtx(addx(mulx(gx, gx), mulx(gy, gy)))));
    } break;
    default: return stencil_epilogue(op, n, s);
  }
  return clamp01(v);
}

}  // namespace vrgdg

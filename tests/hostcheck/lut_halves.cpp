// lut_halves.cpp — TEST INFRASTRUCTURE for tests/test_hostcheck_lut_halves.py.  Compiled with g++ -ffp-contract=off like
// hostcheck.cpp.  Checks that the split evaluation of a LUT cell (lut_half / lut_combine, lutp_half / lutp_combine on cells whose
// sectors hold corner or coefficient XYZ in slot 4X + 2Y + Z) is bit-identical to a whole-sector evaluation written against the
// other natural slot order, X + 2Y + 4Z, with the operation tree of the trilinear interpolation (VRGDG_IV_Adjustments.py:318-339)
// and of the Horner form spelt out corner by corner.
#include "../../comfyui-vrgamedevgirl_b200/csrc/vrgdg_math.cuh"
#include <stdint.h>
#include <string.h>

using namespace vrgdg;

namespace {

// corners of cell (b, g, r), channel ch, corner cXYZ at index X + 2Y + 4Z
void ref_corners(const float* lut3, int S, int b, int g, int r, int ch, float* c) {
  const int b1 = (b + 1 < S) ? b + 1 : S - 1, g1 = (g + 1 < S) ? g + 1 : S - 1, r1 = (r + 1 < S) ? r + 1 : S - 1;
  for (int k = 0; k < 8; ++k) {
    const int rr = (k & 1) ? r1 : r, gg = (k & 2) ? g1 : g, bb = (k & 4) ? b1 : b;
    c[k] = lut3[((size_t)(bb * S + gg) * S + rr) * 3 + ch];
  }
}

// coefficients k_XYZ at index X + 2Y + 4Z: differences along r, then g, then b, in double, rounded once
void ref_coefficients(const float* c, float* kf) {
  double k[8];
  for (int i = 0; i < 8; ++i) k[i] = (double)c[i];
  for (int bit = 1; bit < 8; bit <<= 1)
    for (int i = 0; i < 8; ++i) if (i & bit) k[i] -= k[i ^ bit];
  for (int i = 0; i < 8; ++i) kf[i] = (float)k[i];
}

template <bool EXACT>
float ref_channel(const float* c, float fr, float fg, float fb) {
  const float omr = subx(1.0f, fr), omg = subx(1.0f, fg), omb = subx(1.0f, fb);
  const float c00 = lerp_ref<EXACT>(c[0], c[4], fb, omb), c01 = lerp_ref<EXACT>(c[2], c[6], fb, omb);
  const float c10 = lerp_ref<EXACT>(c[1], c[5], fb, omb), c11 = lerp_ref<EXACT>(c[3], c[7], fb, omb);
  return clamp01(lerp_ref<EXACT>(lerp_ref<EXACT>(c00, c01, fg, omg), lerp_ref<EXACT>(c10, c11, fg, omg), fr, omr));
}

float ref_poly(const float* k, float fr, float fg, float fb) {
  const float a0 = fmaf(fb, k[4], k[0]), b0 = fmaf(fb, k[5], k[1]);
  const float a1 = fmaf(fb, k[6], k[2]), b1 = fmaf(fb, k[7], k[3]);
  return clamp01(fmaf(fr, fmaf(fg, b1, b0), fmaf(fg, a1, a0)));
}

int differ(float a, float b) { uint32_t x, y; memcpy(&x, &a, 4); memcpy(&y, &b, 4); return x != y; }

}  // namespace

extern "C" {

// Every cell of the [S][S][S][3] table `lut3` at each of the n fraction triples `f` ([n][3]: fr, fg, fb); returns the number of
// mismatches (packed slots, exact / contracted corner form, coefficient form, each through lut_channel / lutp_channel and through
// the two halves) and stores the number of comparisons in *checked.
int64_t lh_check(const float* lut3, int S, const float* f, int n, int64_t* checked) {
  int64_t bad = 0, total = 0;
  float cell[LUT_CELL_FLOATS], poly[LUT_CELL_FLOATS];
  for (int b = 0; b < S; ++b) for (int g = 0; g < S; ++g) for (int r = 0; r < S; ++r) {
    lut_pack_entry(lut3, S, b, g, r, cell);
    lutp_pack_entry(lut3, S, b, g, r, poly);
    for (int ch = 0; ch < 3; ++ch) {
      float c[8], k[8];
      ref_corners(lut3, S, b, g, r, ch, c);
      ref_coefficients(c, k);
      const float* q = cell + 8 * ch;
      const float* p = poly + 8 * ch;
      for (int i = 0; i < 8; ++i) {               // index X + 2Y + 4Z -> slot 4X + 2Y + Z
        const int slot = 4 * (i & 1) + (i & 2) + (i >> 2);
        bad += differ(q[slot], c[i]) + differ(p[slot], k[i]);
        total += 2;
      }
      F8 q8, p8;
      for (int i = 0; i < 8; ++i) { q8.v[i] = q[i]; p8.v[i] = p[i]; }
      for (int j = 0; j < n; ++j) {
        const float fr = f[3 * j], fg = f[3 * j + 1], fb = f[3 * j + 2];
        const float omr = subx(1.0f, fr), omg = subx(1.0f, fg), omb = subx(1.0f, fb);
        const float want_x = ref_channel<true>(c, fr, fg, fb), want_f = ref_channel<false>(c, fr, fg, fb), want_p = ref_poly(k, fr, fg, fb);
        bad += differ(lut_channel<true>(q8, fr, fg, fb, omr, omg, omb), want_x);
        bad += differ(lut_combine<true>(lut_half<true>(q, fg, fb, omg, omb), lut_half<true>(q + 4, fg, fb, omg, omb), fr, omr), want_x);
        bad += differ(lut_channel<false>(q8, fr, fg, fb, omr, omg, omb), want_f);
        bad += differ(lut_combine<false>(lut_half<false>(q, fg, fb, omg, omb), lut_half<false>(q + 4, fg, fb, omg, omb), fr, omr), want_f);
        bad += differ(lutp_channel(p8, fr, fg, fb), want_p);
        bad += differ(lutp_combine(lutp_half(p, fg, fb), lutp_half(p + 4, fg, fb), fr), want_p);
        total += 6;
      }
    }
  }
  *checked = total;
  return bad;
}

}  // extern "C"

// vrgdg_resize.cuh — the resample step either side of the enhancer (_resize_batch / _restore_batch,
// VRGDG_VideoEnhanceNodes.py:54-106) and the restore blend (VRGDG_VideoEnhanceNodes.py:408-414).
//
// One kernel covers every fit mode: a source ROI is resampled to res_w x res_h (F.interpolate semantics, align_corners=False,
// size= given so scale = in / out in fp32) and output pixel (x, y) shows resampled pixel (x - off_x, y - off_y); pixels that
// fall outside the resampled image are 0 (the letterbox bars).  "Stretch" has off = 0 and res = target, "Crop to fill" a negative
// offset, "Fit with letterbox" a positive one, "restore" a ROI.  The result is clamped to [0,1] like the reference's.
//
//   nearest : src = min(floor(dst * scale), in - 1)  (ATen "nearest", identity / exact-2x shortcuts give the same indices)
//   bilinear: src = max(scale * (dst + 0.5) - 0.5, 0), two taps per axis
//   bicubic : src = scale * (dst + 0.5) - 0.5, Keys kernel A = -0.75, four border-clamped taps per axis
//   area    : adaptive average over [o*in / out, ((o+1)*in + out - 1) / out), i.e. floor(o*in/out) .. ceil((o+1)*in/out) in exact
//             int64 arithmetic (ATen's start_index / end_index), summed in row-major order, then / rows / cols
//
// Nearest and area are bit-identical to torch; bilinear / bicubic agree to fp32 rounding (ATen picks between two differently
// associated CPU kernels depending on the thread count, so "the" reference bit pattern is not defined; tests use 2e-6).
// Bound: HBM on the larger side (write side when upscaling) — a gather through L1 with warp-coherent addresses.
#pragma once
#include "vrgdg_b200.h"
#include "vrgdg_kernels.cuh"

namespace vrgdg {

struct ResizeParams {
  int B, Hs, Ws, Cs;        // source frames [B,Hs,Ws,Cs], Cs = 3 or 4 (alpha ignored)
  int Ht, Wt;               // output frames [B,Ht,Wt,3]
  int mode;                 // VRGDG_RESIZE_*
  int x0, y0, sw, sh;       // ROI
  int rw, rh;               // resampled size
  int ox, oy;               // placement
  float scale_x, scale_y;   // (float)sw / rw, (float)sh / rh
};

__device__ __forceinline__ void cubic_weights(float t, float w[4]) {
  const float A = -0.75f;
  const float x0 = t + 1.0f, x1 = t, x2 = 1.0f - t, x3 = 2.0f - t;
  w[0] = ((A * x0 - 5.0f * A) * x0 + 8.0f * A) * x0 - 4.0f * A;
  w[1] = ((A + 2.0f) * x1 - (A + 3.0f)) * x1 * x1 + 1.0f;
  w[2] = ((A + 2.0f) * x2 - (A + 3.0f)) * x2 * x2 + 1.0f;
  w[3] = ((A * x3 - 5.0f * A) * x3 + 8.0f * A) * x3 - 4.0f * A;
}

template <typename T>
__device__ __forceinline__ void px_ld(const T* __restrict__ p, float v[3]) {
  v[0] = Elem<T>::ld(__ldg(p)); v[1] = Elem<T>::ld(__ldg(p + 1)); v[2] = Elem<T>::ld(__ldg(p + 2));
}

// Resampled pixel (x, y) of one source frame (frame = its first element) in fp32, before the clamp: the arithmetic of every fit
// mode, shared by k_resize and k_restore so that the two cannot drift apart.  0 outside the resampled image (letterbox bars).
template <typename T, int MODE>
__device__ __forceinline__ void resample_px(const T* __restrict__ frame, const ResizeParams& R, int x, int y, float o[3]) {
  o[0] = o[1] = o[2] = 0.0f;
  const int rx = x - R.ox, ry = y - R.oy;
  if (rx >= 0 && rx < R.rw && ry >= 0 && ry < R.rh) {
    const T* src = frame + (int64_t)R.y0 * R.Ws * R.Cs + (int64_t)R.x0 * R.Cs;
    const int64_t rs = (int64_t)R.Ws * R.Cs;   // row stride in elements
    if (MODE == VRGDG_RESIZE_NEAREST) {
      const int sx = min((int)floorf(mulx((float)rx, R.scale_x)), R.sw - 1);
      const int sy = min((int)floorf(mulx((float)ry, R.scale_y)), R.sh - 1);
      px_ld(src + sy * rs + (int64_t)sx * R.Cs, o);
    } else if (MODE == VRGDG_RESIZE_BILINEAR) {
      const float fx = fmaxf(R.scale_x * ((float)rx + 0.5f) - 0.5f, 0.0f);
      const float fy = fmaxf(R.scale_y * ((float)ry + 0.5f) - 0.5f, 0.0f);
      const int ix = min((int)fx, R.sw - 1), iy = min((int)fy, R.sh - 1);
      const float lx = fminf(fmaxf(fx - (float)ix, 0.0f), 1.0f), ly = fminf(fmaxf(fy - (float)iy, 0.0f), 1.0f);
      const int ix1 = min(ix + 1, R.sw - 1), iy1 = min(iy + 1, R.sh - 1);
      float p00[3], p01[3], p10[3], p11[3];
      px_ld(src + iy * rs + (int64_t)ix * R.Cs, p00);
      px_ld(src + iy * rs + (int64_t)ix1 * R.Cs, p01);
      px_ld(src + iy1 * rs + (int64_t)ix * R.Cs, p10);
      px_ld(src + iy1 * rs + (int64_t)ix1 * R.Cs, p11);
      const float wx0 = 1.0f - lx, wy0 = 1.0f - ly;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float r0 = fmaf(p01[c], lx, p00[c] * wx0), r1 = fmaf(p11[c], lx, p10[c] * wx0);
        o[c] = fmaf(r1, ly, r0 * wy0);
      }
    } else if (MODE == VRGDG_RESIZE_BICUBIC) {
      const float fx = R.scale_x * ((float)rx + 0.5f) - 0.5f, fy = R.scale_y * ((float)ry + 0.5f) - 0.5f;
      const float flx = floorf(fx), fly = floorf(fy);
      const int ix = (int)flx, iy = (int)fly;
      float wx[4], wy[4];
      cubic_weights(fx - flx, wx);
      cubic_weights(fy - fly, wy);
      int xs[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) xs[k] = max(min(ix - 1 + k, R.sw - 1), 0) * R.Cs;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const T* row = src + (int64_t)max(min(iy - 1 + j, R.sh - 1), 0) * rs;
        float a[3] = {0.0f, 0.0f, 0.0f};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float p[3];
          px_ld(row + xs[k], p);
#pragma unroll
          for (int c = 0; c < 3; ++c) a[c] = fmaf(p[c], wx[k], a[c]);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c] = fmaf(a[c], wy[j], o[c]);
      }
    } else {   // area: ATen's integer window bounds (an fp32 quotient rounds once o*in passes 2^24 and picks the wrong window)
      const int xa = (int)(((int64_t)rx * R.sw) / R.rw);
      const int xb = (int)(((int64_t)(rx + 1) * R.sw + R.rw - 1) / R.rw);
      const int ya = (int)(((int64_t)ry * R.sh) / R.rh);
      const int yb = (int)(((int64_t)(ry + 1) * R.sh + R.rh - 1) / R.rh);
      for (int yy = ya; yy < yb; ++yy) {
        const T* row = src + yy * rs;
        for (int xx = xa; xx < xb; ++xx) {
          float p[3];
          px_ld(row + (int64_t)xx * R.Cs, p);
#pragma unroll
          for (int c = 0; c < 3; ++c) o[c] = addx(o[c], p[c]);
        }
      }
      const float kh = (float)(yb - ya), kw = (float)(xb - xa);    // ATen: scalar_t(sum / kh / kw), two roundings
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c] = divx(divx(o[c], kh), kw);
    }
  }
}

template <typename T, int MODE>
__global__ void __launch_bounds__(256) k_resize(const T* __restrict__ in, T* __restrict__ out, const ResizeParams R) {
  const int64_t total = (int64_t)R.B * R.Ht * R.Wt;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % R.Wt);
    const int64_t q = i / R.Wt;
    const int y = (int)(q % R.Ht);
    const int b = (int)(q / R.Ht);
    float o[3];
    resample_px<T, MODE>(in + (int64_t)b * R.Hs * R.Ws * R.Cs, R, x, y, o);
    T* dst = out + i * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) dst[c] = Elem<T>::st(clamp01(o[c]));
  }
}

// restored * s + originals * (1 - s), clamped (VRGDG_VideoEnhanceNodes.py:408-414; (1 - s) is formed in double by Python and
// rounded once, which the caller does)
template <typename T>
__global__ void __launch_bounds__(256) k_blend(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ out, int64_t n,
                                               float wa, float wb) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = Elem<T>::st(clamp01(addx(mulx(Elem<T>::ld(a[i]), wa), mulx(Elem<T>::ld(b[i]), wb))));
}

// The restore node in one pass (VRGDG_VideoEnhanceNodes.py:404-418 = _restore_batch, .to(dtype), the blend and the clamp).  For
// output frame b < n_restored and colour channel c < 3:
//   r   = T(clamp01(resample_px(enhanced[b], x, y)[c]))          k_resize's value, rounded to the frame type as `restored` is
//   out = T(clamp01(orig * w_orig + r * w_restored))             k_blend's expression, one rounding per operation
// every other element (the alpha of RGBA originals, frames past the last enhanced one): out = T(clamp(orig, 0, 1)), NaN kept as
// torch.clamp keeps it.  Originals and output move with 16-byte accesses, PX = 16 / sizeof(T) whole pixels (CO words) per thread,
// when W % PX == 0 and both pointers are 16-byte aligned, else one pixel per thread; the enhanced gather goes through L1 as
// k_resize's does.  Algorithmic bytes per output pixel: 2 * CO * sizeof(T) for the originals and the output, plus the enhanced
// frame's share, He * We * Ce * sizeof(T) / (H * W) for a restored frame.  Bound: HBM.
struct RestoreParams {
  ResizeParams R;           // enhanced frames [n_restored, Hs, Ws, Cs] resampled to the output size Ht x Wt
  int B, Co;                // originals and output [B, Ht, Wt, Co], Co = 3 or 4
  int n_restored;           // frames [0, n_restored) are blended, the rest only clamped
  float w_orig, w_restored;
};

__device__ __forceinline__ float clamp01_keep_nan(float v) { return v != v ? v : clamp01(v); }

template <typename T, int MODE, int CO, bool VEC>
__global__ void __launch_bounds__(256) k_restore(const T* __restrict__ enh, const T* __restrict__ orig, T* __restrict__ out,
                                                 const RestoreParams P) {
  constexpr int PX = VEC ? (int)(16 / sizeof(T)) : 1;
  constexpr int NE = PX * CO;
  const ResizeParams& R = P.R;
  const int gw = R.Wt / PX;                                   // pixel groups per row
  const int64_t total = (int64_t)P.B * R.Ht * gw;
  const int64_t enh_frame = (int64_t)R.Hs * R.Ws * R.Cs;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x0 = (int)(i % gw) * PX;
    const int64_t q = i / gw;                                 // b * Ht + y
    const int y = (int)(q % R.Ht);
    const int b = (int)(q / R.Ht);
    const int64_t e0 = (q * R.Wt + x0) * CO;
    union { uint4 w[CO]; T e[16 / sizeof(T) * CO]; } u;     // the scalar path uses the first CO elements
    if (VEC) {
#pragma unroll
      for (int k = 0; k < CO; ++k) u.w[k] = __ldg(reinterpret_cast<const uint4*>(orig + e0) + k);
    } else {
#pragma unroll
      for (int k = 0; k < NE; ++k) u.e[k] = __ldg(orig + e0 + k);
    }
    if (b < P.n_restored) {
      const T* ef = enh + (int64_t)b * enh_frame;
#pragma unroll
      for (int p = 0; p < PX; ++p) {
        float r[3];
        resample_px<T, MODE>(ef, R, x0 + p, y, r);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float rv = Elem<T>::ld(Elem<T>::st(clamp01(r[c])));
          const float ov = Elem<T>::ld(u.e[p * CO + c]);
          u.e[p * CO + c] = Elem<T>::st(clamp01(addx(mulx(ov, P.w_orig), mulx(rv, P.w_restored))));
        }
        if (CO == 4) u.e[p * CO + 3] = Elem<T>::st(clamp01_keep_nan(Elem<T>::ld(u.e[p * CO + 3])));
      }
    } else {
#pragma unroll
      for (int k = 0; k < NE; ++k) u.e[k] = Elem<T>::st(clamp01_keep_nan(Elem<T>::ld(u.e[k])));
    }
    if (VEC) {
#pragma unroll
      for (int k = 0; k < CO; ++k) reinterpret_cast<uint4*>(out + e0)[k] = u.w[k];
    } else {
#pragma unroll
      for (int k = 0; k < NE; ++k) out[e0 + k] = u.e[k];
    }
  }
}

template <typename T, int MODE, int CO, bool VEC>
static cudaError_t launch_restore_k(const T* enh, const T* orig, T* out, const RestoreParams& P, const LaunchCtx& ctx) {
  constexpr int PX = VEC ? (int)(16 / sizeof(T)) : 1;
  const int64_t groups = (int64_t)P.B * P.R.Ht * (P.R.Wt / PX);
  const int grid = (int)std::min<int64_t>((groups + 255) / 256, (int64_t)ctx.sms * 32);
  k_restore<T, MODE, CO, VEC><<<grid, 256, 0, ctx.stream>>>(enh, orig, out, P);
  count_launch();
  return cudaGetLastError();
}

template <typename T, int MODE>
static cudaError_t launch_restore_m(const T* enh, const T* orig, T* out, const RestoreParams& P, bool vec, const LaunchCtx& ctx) {
  if (P.Co == 3) return vec ? launch_restore_k<T, MODE, 3, true>(enh, orig, out, P, ctx) : launch_restore_k<T, MODE, 3, false>(enh, orig, out, P, ctx);
  return vec ? launch_restore_k<T, MODE, 4, true>(enh, orig, out, P, ctx) : launch_restore_k<T, MODE, 4, false>(enh, orig, out, P, ctx);
}

template <typename T>
cudaError_t launch_restore(const void* enh, const void* orig, void* out, const RestoreParams& P, const LaunchCtx& ctx) {
  if constexpr (sizeof(T) == 1) {
    return cudaErrorInvalidValue;                             // float frames only (the ABI refuses uint8 before this)
  } else {
    if ((int64_t)P.B * P.R.Ht * P.R.Wt == 0) return cudaSuccess;
    constexpr int PX = (int)(16 / sizeof(T));
    const bool vec = P.R.Wt % PX == 0 && ((reinterpret_cast<uintptr_t>(orig) | reinterpret_cast<uintptr_t>(out)) & 15u) == 0;
    const T* te = reinterpret_cast<const T*>(enh);
    const T* to = reinterpret_cast<const T*>(orig);
    T* tout = reinterpret_cast<T*>(out);
    switch (P.R.mode) {
      case VRGDG_RESIZE_NEAREST: return launch_restore_m<T, VRGDG_RESIZE_NEAREST>(te, to, tout, P, vec, ctx);
      case VRGDG_RESIZE_BILINEAR: return launch_restore_m<T, VRGDG_RESIZE_BILINEAR>(te, to, tout, P, vec, ctx);
      case VRGDG_RESIZE_BICUBIC: return launch_restore_m<T, VRGDG_RESIZE_BICUBIC>(te, to, tout, P, vec, ctx);
      default: return launch_restore_m<T, VRGDG_RESIZE_AREA>(te, to, tout, P, vec, ctx);
    }
  }
}

template <typename T>
cudaError_t launch_resize(const void* in, void* out, const ResizeParams& R, const LaunchCtx& ctx) {
  const int64_t total = (int64_t)R.B * R.Ht * R.Wt;
  if (total == 0) return cudaSuccess;
  const int grid = (int)std::min<int64_t>((total + 255) / 256, (int64_t)ctx.sms * 32);
  const T* tin = reinterpret_cast<const T*>(in);
  T* tout = reinterpret_cast<T*>(out);
  switch (R.mode) {
    case VRGDG_RESIZE_NEAREST: k_resize<T, VRGDG_RESIZE_NEAREST><<<grid, 256, 0, ctx.stream>>>(tin, tout, R); break;
    case VRGDG_RESIZE_BILINEAR: k_resize<T, VRGDG_RESIZE_BILINEAR><<<grid, 256, 0, ctx.stream>>>(tin, tout, R); break;
    case VRGDG_RESIZE_BICUBIC: k_resize<T, VRGDG_RESIZE_BICUBIC><<<grid, 256, 0, ctx.stream>>>(tin, tout, R); break;
    default: k_resize<T, VRGDG_RESIZE_AREA><<<grid, 256, 0, ctx.stream>>>(tin, tout, R); break;
  }
  count_launch();
  return cudaGetLastError();
}

template <typename T>
cudaError_t launch_blend(const void* a, const void* b, void* out, int64_t n, float wa, float wb, const LaunchCtx& ctx) {
  if (n == 0) return cudaSuccess;
  const int grid = (int)std::min<int64_t>((n + 255) / 256, (int64_t)ctx.sms * 32);
  k_blend<T><<<grid, 256, 0, ctx.stream>>>(reinterpret_cast<const T*>(a), reinterpret_cast<const T*>(b), reinterpret_cast<T*>(out), n, wa, wb);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vrgdg

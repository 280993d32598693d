// vrgdg_inst.cuh — host launchers, instantiated once per frame dtype (vrgdg_f32.cu / _f16.cu / _bf16.cu)
#pragma once
#include "vrgdg_kernels.cuh"
#include <algorithm>
#include "vrgdg_adjust.cuh"
#include "vrgdg_resize.cuh"
#include "vrgdg_temporal.cuh"
#include "vrgdg_histmatch.cuh"
#include <string.h>
#include <stdlib.h>

namespace vrgdg {

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

template <typename K>
static int occupancy_of(K kernel, int threads, size_t smem) {
  int occ = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, threads, smem) != cudaSuccess || occ < 1) occ = 1;
  return occ;
}

// ---- k_point ---------------------------------------------------------------------------------
template <typename T, int MASK, bool EXACT, bool VEC>
static cudaError_t launch_point_k(const void* in, void* out, const PointParams& P, const LaunchCtx& ctx) {
  constexpr int PX = VEC ? (int)(3 * sizeof(typename Io<T>::word_t) / (3 * sizeof(T))) : 1;
  const int64_t groups = (P.hw + PX - 1) / PX;
  const int bpf = (int)((groups + 255) / 256);
  const int64_t total = (int64_t)bpf * P.B;
  if (total == 0) return cudaSuccess;
  auto kern = k_point<T, MASK, EXACT, VEC>;
  if (MASK & ST_LUT) cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 0);   // all of it as L1 for the gather
  static int occ = occupancy_of(kern, 256, 0);
  const int64_t cap = (int64_t)ctx.sms * occ * 4;
  const int grid = (int)std::min<int64_t>(total, cap);
  kern<<<grid, 256, 0, ctx.stream>>>(reinterpret_cast<const T*>(in), reinterpret_cast<T*>(out), P, bpf, total);
  count_launch();
  return cudaGetLastError();
}

template <typename T, int MASK, bool EXACT>
static cudaError_t launch_point_v(const void* in, void* out, const PointParams& P, const LaunchCtx& ctx) {
  typedef typename Io<T>::word_t word_t;
  constexpr int PX = (int)(3 * sizeof(word_t) / (3 * sizeof(T)));
  auto ok = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & (sizeof(word_t) - 1)) == 0; };
  bool vec = (P.hw % PX == 0) && (P.W % PX == 0) && ok(in) && ok(out) &&
             (!(MASK & ST_GRAIN) || P.ext_noise == nullptr || aligned16(P.ext_noise));
  if (vec) return launch_point_k<T, MASK, EXACT, true>(in, out, P, ctx);
  return launch_point_k<T, MASK, EXACT, false>(in, out, P, ctx);
}

template <typename T>
cudaError_t launch_point(const void* in, void* out, const PointParams& P, int mask, bool exact, const LaunchCtx& ctx) {
  // masks without grain have no inexact variant (colour match always rounds like the reference; LUT alone is exact)
#define VRGDG_PT(M)                                                                    \
  case M:                                                                              \
    if constexpr (((M) & ST_GRAIN) != 0) {                                             \
      if (!exact) return launch_point_v<T, M, false>(in, out, P, ctx);                 \
    }                                                                                  \
    return launch_point_v<T, M, true>(in, out, P, ctx);
  switch (mask) {
    VRGDG_PT(1) VRGDG_PT(2) VRGDG_PT(3) VRGDG_PT(4) VRGDG_PT(5) VRGDG_PT(6) VRGDG_PT(7)
    case ST_CMF:                 // second pass of the f-plane schedule: input = (fx, fy, fz) planes, fp32 only
      if constexpr (sizeof(T) == 4) return launch_point_v<T, ST_CMF, true>(in, out, P, ctx);
      return cudaErrorInvalidValue;
    case ST_CMF | ST_LUT:
      if constexpr (sizeof(T) == 4) {
        if (!exact) return launch_point_v<T, ST_CMF | ST_LUT, false>(in, out, P, ctx);
        return launch_point_v<T, ST_CMF | ST_LUT, true>(in, out, P, ctx);
      }
      return cudaErrorInvalidValue;
    default: return cudaErrorInvalidValue;
  }
#undef VRGDG_PT
}

template <typename T>
cudaError_t launch_lut_rgba(const void* in, void* out, int64_t npix, const LutParams& L, const LaunchCtx& ctx) {
  if (npix == 0) return cudaSuccess;
  const int grid = (int)std::min<int64_t>((npix + 255) / 256, (int64_t)ctx.sms * 32);
  k_lut_rgba<T><<<grid, 256, 0, ctx.stream>>>(reinterpret_cast<const T*>(in), reinterpret_cast<T*>(out), npix, L);
  count_launch();
  return cudaGetLastError();
}

// ---- k_tile ------------------------------------------------------------------------------------
template <typename T>
void tile_geometry(int H, int RW, int& tiles_x, int& tiles_y, int& box_x, int& box_y) {
  using C = TileCfg<T, 0>;         // tile geometry is the same for every configuration
  tiles_x = (RW + C::TXE - 1) / C::TXE;
  tiles_y = (H + C::TY - 1) / C::TY;
  box_x = C::BX;
  box_y = C::ROWS;
}

template <typename T, int MASK, bool EXACT, int CH = 3>
static cudaError_t launch_tile_k(const CUtensorMap* tmap, const void* in, void* out, TileParams& Q, const LaunchCtx& ctx) {
  auto kern = k_tile<T, MASK, EXACT, CH>;
  constexpr size_t smem = tile_smem_bytes<T, MASK, CH>();
  // per device context, so set on every launch (single-process multi-GPU hosts)
  cudaError_t attr = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (attr != cudaSuccess) return attr;
  constexpr int NT = TileCfg<T, MASK, CH>::THREADS;
  if (MASK & ST_LUT) cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, (int)((smem + 1024) * TileCfg<T, MASK, CH>::MINB * 100 / (228 * 1024)) + 1);
  static int occ = occupancy_of(kern, NT, smem);
  if (Q.total_tiles == 0) return cudaSuccess;
  const int grid = (int)std::min<int64_t>(Q.total_tiles, (int64_t)ctx.sms * occ);
  CUtensorMap dummy;
  if (!tmap) { memset(&dummy, 0, sizeof(dummy)); tmap = &dummy; }
  kern<<<grid, NT, smem, ctx.stream>>>(*tmap, reinterpret_cast<const T*>(in), reinterpret_cast<T*>(out), Q);
  count_launch();
  return cudaGetLastError();
}

template <typename T>
cudaError_t launch_tile(const CUtensorMap* tmap, const void* in, void* out, TileParams& Q, int mask, bool exact,
                        const LaunchCtx& ctx) {
#define VRGDG_TL(M)                                                                        \
  case M:                                                                                  \
    if constexpr (((M) & ST_GRAIN) != 0) {                                                 \
      if (!exact) return launch_tile_k<T, M, false>(tmap, in, out, Q, ctx);                \
    }                                                                                      \
    return launch_tile_k<T, M, true>(tmap, in, out, Q, ctx);
  switch (mask) {
    VRGDG_TL(0) VRGDG_TL(1) VRGDG_TL(2) VRGDG_TL(3) VRGDG_TL(4) VRGDG_TL(5) VRGDG_TL(6) VRGDG_TL(7)
    VRGDG_TL(8)     // stencil + post grain staged in a shared-memory plane (the enhancer chain)
    case ST_CMF:
      if constexpr (sizeof(T) == 4) return launch_tile_k<T, ST_CMF, true>(tmap, in, out, Q, ctx);
      return cudaErrorInvalidValue;
    case ST_CMF | ST_LUT:
      if constexpr (sizeof(T) == 4) {
        if (!exact) return launch_tile_k<T, ST_CMF | ST_LUT, false>(tmap, in, out, Q, ctx);
        return launch_tile_k<T, ST_CMF | ST_LUT, true>(tmap, in, out, Q, ctx);
      }
      return cudaErrorInvalidValue;
    default: return cudaErrorInvalidValue;
  }
#undef VRGDG_TL
}

// plain 3x3 stencil on RGBA frames (Q.RW = 4*W), read interleaved as stored.  The NumPy-path ops only: the torch paths (ops 3 and 5)
// convolve with groups=3 and reject 4 channels in the reference.  Exact arithmetic on fp32 frames, the fast variant on 16-bit ones,
// as vrgdg_stencil3x3 does, so that every channel equals the 3-channel kernel's result bit for bit.  Byte frames are 3-channel BGR.
template <typename T>
cudaError_t launch_tile_rgba(const CUtensorMap* tmap, const void* in, void* out, TileParams& Q, const LaunchCtx& ctx) {
  if constexpr (sizeof(T) == 1) {
    return cudaErrorInvalidValue;
  } else {
    switch (Q.op) {
      case 1: case 2: case 4:
        if constexpr (sizeof(T) == 4) {
          if (Q.exact_stencil) return launch_tile_k<T, 0, true, 4>(tmap, in, out, Q, ctx);
        } else {
          if (!Q.exact_stencil) return launch_tile_k<T, 0, false, 4>(tmap, in, out, Q, ctx);
        }
        return cudaErrorInvalidValue;
      default: return cudaErrorInvalidValue;
    }
  }
}

// 3D LUT then 3x3 stencil on RGBA frames in one tile pass (Q.RW = 4*W, Q.P.lut filled): RGB graded, alpha carried as k_lut_rgba
// carries it, every channel then filtered.  The LUT is the exact one of the 3-channel chain (no grain draws noise here); the stencil
// arithmetic follows launch_tile_rgba's rule, exact on fp32 frames and fast on 16-bit ones, so that the RGB channels equal the
// 3-channel fused chain's bit for bit.  NumPy-path ops only; byte frames are 3-channel BGR.
template <typename T>
cudaError_t launch_tile_rgba_lut(const CUtensorMap* tmap, const void* in, void* out, TileParams& Q, const LaunchCtx& ctx) {
  if constexpr (sizeof(T) == 1) {
    return cudaErrorInvalidValue;
  } else {
    switch (Q.op) {
      case 1: case 2: case 4:
        if constexpr (sizeof(T) == 4) {
          if (Q.exact_stencil) return launch_tile_k<T, ST_LUT, true, 4>(tmap, in, out, Q, ctx);
        } else {
          if (!Q.exact_stencil) return launch_tile_k<T, ST_LUT, true, 4>(tmap, in, out, Q, ctx);
        }
        return cudaErrorInvalidValue;
      default: return cudaErrorInvalidValue;
    }
  }
}

// ---- moments -------------------------------------------------------------------------------------
template <typename T, bool GRAIN, bool VEC, int NT>
static cudaError_t launch_moments_k(const T* src, const PointParams& P, int row0, int rows, double* partials, float* fplanes, const LaunchCtx& ctx) {
  auto kern = k_lab_moments<T, GRAIN, VEC, NT>;
  if (NT == MOMENT_UNIT) {
    // pipelined schedule: these blocks share SMs with two resident k_tile CTAs, whose shared-memory carve-out they must not fight
    // (an SM changes its carve-out only when idle, which would serialise the two kernels)
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 64);
  }
  dim3 grid(MOMENT_BLOCKS / (NT / MOMENT_UNIT), P.B);
  kern<<<grid, NT, 0, ctx.stream>>>(src, P, row0, rows, partials, fplanes);
  count_launch();
  return cudaGetLastError();
}

template <typename T>
cudaError_t launch_moments(const void* in, const PointParams& P, bool grain, int row0, int rows, double* sums,
                           double* partials, const LaunchCtx& ctx, float* fplanes, bool small_blocks) {
  if (P.B == 0) return cudaSuccess;
  typedef typename Io<T>::word_t word_t;
  constexpr int PX = (int)(sizeof(word_t) / sizeof(T));
  const bool vec = (P.W % PX == 0) && ((reinterpret_cast<uintptr_t>(in) & (sizeof(word_t) - 1)) == 0);
  if (fplanes && !(vec && sizeof(T) == 4 && aligned16(fplanes))) return cudaErrorInvalidValue;   // the ABI layer only asks for planes when this holds
  const T* src = reinterpret_cast<const T*>(in);
  cudaError_t e;
  if (small_blocks && vec && grain) e = launch_moments_k<T, true, true, MOMENT_UNIT>(src, P, row0, rows, partials, fplanes, ctx);
  else if (small_blocks && vec) e = launch_moments_k<T, false, true, MOMENT_UNIT>(src, P, row0, rows, partials, fplanes, ctx);
  else if (grain && vec) e = launch_moments_k<T, true, true, 256>(src, P, row0, rows, partials, fplanes, ctx);
  else if (grain) e = launch_moments_k<T, true, false, 256>(src, P, row0, rows, partials, fplanes, ctx);
  else if (vec) e = launch_moments_k<T, false, true, 256>(src, P, row0, rows, partials, fplanes, ctx);
  else e = launch_moments_k<T, false, false, 256>(src, P, row0, rows, partials, fplanes, ctx);
  if (e != cudaSuccess) return e;
  k_moments_final<<<P.B, 32, 0, ctx.stream>>>(partials, MOMENT_BLOCKS, (double)rows * (double)P.W, sums);
  count_launch();
  return cudaGetLastError();
}

// ---- the global generator's noise, materialised --------------------------------------------------------
// float dtypes only (the ABI refuses uint8 frames first); w.rows * T_full / 256 < 2^31 is the ABI's check
template <typename T>
cudaError_t launch_torch_global_noise(void* out, uint64_t seed, uint64_t o0, const TorchGlobalWindow& w, const LaunchCtx& ctx) {
  const uint32_t blocks_full = w.T_full / TORCH_RANDN_BLOCK, total = w.rows * blocks_full;
  if (total == 0) return cudaSuccess;
  auto kern = k_torch_global_noise<T>;
  static int occ = occupancy_of(kern, 256, 0);
  const int grid = (int)std::min<int64_t>(total, (int64_t)ctx.sms * occ);
  kern<<<grid, 256, 0, ctx.stream>>>(reinterpret_cast<T*>(out), seed, o0, w, blocks_full);
  count_launch();
  return cudaGetLastError();
}

// ---- u8 codecs ---------------------------------------------------------------------------------
template <typename T>
cudaError_t launch_u8_in(const uint8_t* in, void* out, int64_t npix, const LaunchCtx& ctx) {
  if (npix == 0) return cudaSuccess;
  const int grid = (int)std::min<int64_t>((npix + 255) / 256, (int64_t)ctx.sms * 32);
  k_u8bgr_to_rgb<T><<<grid, 256, 0, ctx.stream>>>(in, reinterpret_cast<T*>(out), npix);
  count_launch();
  return cudaGetLastError();
}
template <typename T>
cudaError_t launch_u8_out(const void* in, uint8_t* out, int64_t npix, const LaunchCtx& ctx) {
  if (npix == 0) return cudaSuccess;
  const int grid = (int)std::min<int64_t>((npix + 255) / 256, (int64_t)ctx.sms * 32);
  k_rgb_to_u8bgr<T><<<grid, 256, 0, ctx.stream>>>(reinterpret_cast<const T*>(in), out, npix);
  count_launch();
  return cudaGetLastError();
}

#define VRGDG_INSTANTIATE(T)                                                                                              \
  template cudaError_t launch_point<T>(const void*, void*, const PointParams&, int, bool, const LaunchCtx&);              \
  template cudaError_t launch_lut_rgba<T>(const void*, void*, int64_t, const LutParams&, const LaunchCtx&);               \
  template cudaError_t launch_tile<T>(const CUtensorMap*, const void*, void*, TileParams&, int, bool, const LaunchCtx&);  \
  template cudaError_t launch_tile_rgba<T>(const CUtensorMap*, const void*, void*, TileParams&, const LaunchCtx&);        \
  template cudaError_t launch_tile_rgba_lut<T>(const CUtensorMap*, const void*, void*, TileParams&, const LaunchCtx&);    \
  template cudaError_t launch_moments<T>(const void*, const PointParams&, bool, int, int, double*, double*, const LaunchCtx&, float*, bool); \
  template cudaError_t launch_adjust<T>(const void*, void*, const AdjustParams&, int, float*, float*, const LaunchCtx&);              \
  template cudaError_t launch_resize<T>(const void*, void*, const ResizeParams&, const LaunchCtx&);                       \
  template cudaError_t launch_blend<T>(const void*, const void*, void*, int64_t, float, float, const LaunchCtx&);         \
  template cudaError_t launch_restore<T>(const void*, const void*, void*, const RestoreParams&, const LaunchCtx&);        \
  template cudaError_t launch_temporal<T>(const void*, void*, const TemporalParams&, const LaunchCtx&);                   \
  template cudaError_t launch_hist_counts<T>(const void*, int, int, int, int, int, uint32_t*, const LaunchCtx&);          \
  template cudaError_t launch_histmatch_apply<T>(const void*, void*, int, int64_t, const float2*, float, float, const LaunchCtx&); \
  template void tile_geometry<T>(int, int, int&, int&, int&, int&);

#define VRGDG_INSTANTIATE_CODECS(T)                                                                                       \
  template cudaError_t launch_u8_in<T>(const uint8_t*, void*, int64_t, const LaunchCtx&);                                 \
  template cudaError_t launch_u8_out<T>(const void*, uint8_t*, int64_t, const LaunchCtx&);

// float frame dtypes only: launchers with no uint8 counterpart
#define VRGDG_INSTANTIATE_FLOAT(T)                                                                                        \
  template cudaError_t launch_torch_global_noise<T>(void*, uint64_t, uint64_t, const TorchGlobalWindow&, const LaunchCtx&);

}  // namespace vrgdg

// vrgdg_kernels.cuh — sm_90a kernels of the post-processing hot path.
//
// Two kernel families cover every entry point of include/vrgdg_b200.h:
//   k_point : streaming per-pixel chain  [grain][colour match][3D LUT]          (no neighbourhood)
//   k_tile  : TMA-staged halo tiles      [grain][colour match][3D LUT] -> 3x3 stencil -> [post grain]
// plus the LAB moment reduction and the uint8 wire-format codecs.
// Data layout: frames [B][H][W][3] channel-fastest; a frame row is RW = 3*W contiguous elements.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include "vrgdg_math.cuh"

namespace vrgdg {

enum {
  ST_GRAIN = 1, ST_CM = 2, ST_LUT = 4,
  ST_POST = 8,   /* k_tile only: post-grain values staged in a shared-memory plane */
  ST_CMF = 16,   /* colour match whose input is NOT rgb but the (fx, fy, fz) planes the moments pass stored (fp32 frames only): the
                    second pass of vrgdg_chain_cm_apply neither redraws the grain nor repeats the forward Lab transform */
  ST_PRE = ST_GRAIN | ST_CM | ST_LUT | ST_CMF   /* per-pixel stages that run before the stencil */
};

// ---- element conversion -------------------------------------------------------------------------
template <typename T> struct Elem;
template <> struct Elem<float> {
  static __device__ __forceinline__ float ld(float v) { return v; }
  static __device__ __forceinline__ float st(float v) { return v; }
};
template <> struct Elem<__half> {
  static __device__ __forceinline__ float ld(__half v) { return __half2float(v); }
  static __device__ __forceinline__ __half st(float v) { return __float2half_rn(v); }
};
template <> struct Elem<__nv_bfloat16> {
  static __device__ __forceinline__ float ld(__nv_bfloat16 v) { return __bfloat162float(v); }
  static __device__ __forceinline__ __nv_bfloat16 st(float v) { return __float2bfloat16_rn(v); }
};

// uint8 frames are the reference's video wire format (cv2 BGR bytes): x/255.0 on the way in, clip(x*255,0,255) TRUNCATED on
// the way out (VRGDG_LUTVideoTools.py:736-752), channel order swapped to RGB inside the kernels.
template <> struct Elem<uint8_t> {
  // v/255.0f, correctly rounded, without the division sequence: q = v*r, q' = fma(fma(-255,q,v), r, q) equals the IEEE quotient
  // for every one of the 256 byte values (checked exhaustively, tests/test_host_logic.py::test_u8_division_identity)
  static __device__ __forceinline__ float ld(uint8_t v) {
    const float r = 1.0f / 255.0f, f = (float)v, q = __fmul_rn(f, r);
    return __fmaf_rn(__fmaf_rn(-255.0f, q, f), r, q);
  }
  static __device__ __forceinline__ uint8_t st(float v) { return (uint8_t)fminf(fmaxf(mulx(v, 255.0f), 0.0f), 255.0f); }
};

template <typename T> struct Io {
  static constexpr bool BGR = false;          // memory order of a pixel's channels
  typedef T noise_t;                          // element type of an external noise tensor
  typedef uint4 word_t;                       // a thread moves 3 words = whole pixels
};
template <> struct Io<uint8_t> {
  static constexpr bool BGR = true;
  typedef float noise_t;
  typedef uint32_t word_t;
};
template <typename T> __device__ __forceinline__ float noise_ld(T v) { return Elem<T>::ld(v); }
template <> __device__ __forceinline__ float noise_ld<float>(float v) { return v; }

// ---- parameters of the per-pixel stages ------------------------------------------------------------
struct PointParams {
  int B, H, W;
  int64_t hw;                  // pixels per frame
  // grain
  float gI, gs, goms;
  uint64_t seed;
  int64_t frame0;
  int seed_mode;
  GrainKey gkey;               // Philox round keys, evaluated on the host
  const void* ext_noise;       // [B,H,W,3] of the frame dtype, or null
  // colour match
  const float* cm_params;      // [B][12]
  float cm_t, cm_omt;
  // LUT
  LutParams lut;
};

#ifndef VRGDG_LUT_POLY
#define VRGDG_LUT_POLY 1             // 0: the fast chains interpolate the corner cells too (A/B switch of tools/build_variant.sh)
#endif

// One pixel through the enabled stages; (zr,zg,zb) = this pixel's N(0,1) triple (generator or external).
template <int MASK, bool EXACT>
__device__ __forceinline__ void process_pixel(const PointParams& P, const CmFold& cmf, float zr, float zg, float zb,
                                              float& r, float& g, float& b) {
  if (MASK & ST_GRAIN) {
    if (EXACT) grain_blend_exact(r, g, b, zr, zg, zb, P.gI, P.gs, P.goms);
    else grain_blend_fast(r, g, b, zr, zg, zb, P.gI, P.gs, P.goms);
  }
  if (MASK & ST_CM) {
    colormatch_fold_pixel(r, g, b, cmf);
  }
  if (MASK & ST_CMF) {
    colormatch_from_f(r, g, b, cmf);          // (r, g, b) hold (fx, fy, fz) on entry
  }
  if (MASK & ST_LUT) {
    float x0 = r, x1 = g, x2 = b;
    if (EXACT || !VRGDG_LUT_POLY) lut3d_eval<EXACT>(P.lut, r, g, b);
    else lutp_eval(P.lut, r, g, b);                  // fast arithmetic: polynomial cells, 7 FMAs per channel
    if (P.lut.blend < 1.0f) {
      r = lut_blend<EXACT>(x0, r, P.lut.blend, P.lut.one_minus_blend);
      g = lut_blend<EXACT>(x1, g, P.lut.blend, P.lut.one_minus_blend);
      b = lut_blend<EXACT>(x2, b, P.lut.blend, P.lut.one_minus_blend);
    }
  }
}

// two pixels at once: all per-pixel stages up to the LUT, then BOTH gathers issued before either is consumed
template <int MASK, bool EXACT>
__device__ __forceinline__ void process_pair(const PointParams& P, const CmFold& cmf, const float* z, float* p) {
  process_pixel<(MASK & ~ST_LUT), EXACT>(P, cmf, z[0], z[1], z[2], p[0], p[1], p[2]);
  process_pixel<(MASK & ~ST_LUT), EXACT>(P, cmf, z[3], z[4], z[5], p[3], p[4], p[5]);
  if (MASK & ST_LUT) {
    float x[6] = {p[0], p[1], p[2], p[3], p[4], p[5]};
    if (EXACT || !VRGDG_LUT_POLY) lut3d_eval2<EXACT>(P.lut, p, p + 3);
    else lutp_eval2(P.lut, p, p + 3);
    if (P.lut.blend < 1.0f) {
#pragma unroll
      for (int i = 0; i < 6; ++i) p[i] = lut_blend<EXACT>(x[i], p[i], P.lut.blend, P.lut.one_minus_blend);
    }
  }
}

// =====================================================================================================
// k_point — streaming chain.  VEC: a thread owns 48 bytes = PX whole pixels (4 fp32 / 8 fp16) moved with
// three 16-byte loads and stores; requires hw % PX == 0 and 16-byte aligned bases.  !VEC: one pixel per
// thread, scalar accesses (any shape / alignment).
// =====================================================================================================
template <typename T, int MASK, bool EXACT, bool VEC>
__global__ void __launch_bounds__(256)
k_point(const T* __restrict__ in, T* __restrict__ out, PointParams P,
        int blocks_per_frame, int64_t total_vblocks) {
  typedef typename Io<T>::word_t word_t;
  typedef typename Io<T>::noise_t noise_t;
  constexpr bool BGR = Io<T>::BGR;
  constexpr int PX = VEC ? (int)(3 * sizeof(word_t) / (3 * sizeof(T))) : 1;   // 4 fp32 / 8 fp16 / 4 u8 pixels; VEC needs W % PX == 0
  constexpr int NE = PX * 3;
  constexpr bool GRAIN = (MASK & ST_GRAIN) != 0;
  const bool has_ext = GRAIN && (P.ext_noise != nullptr);
  for (int64_t vb = blockIdx.x; vb < total_vblocks; vb += gridDim.x) {
    const int frame = (int)(vb / blocks_per_frame);
    const int bif = (int)(vb - (int64_t)frame * blocks_per_frame);
    const int64_t pix0 = ((int64_t)bif * 256 + threadIdx.x) * PX;
    if (pix0 >= P.hw) continue;
    const int64_t e0 = ((int64_t)frame * P.hw + pix0) * 3;
    const GrainFrame gf = grain_frame(P.seed, P.frame0, frame, P.seed_mode);
    CmFold cmf = {};                          // per-frame affine map of the colour match, folded with the strength (uniform per block)
    if (MASK & (ST_CM | ST_CMF)) cmf = cm_fold(P.cm_params + (int64_t)frame * 12, P.cm_t, P.cm_omt);
    const uint32_t y = GRAIN ? (uint32_t)pix0 / (uint32_t)P.W : 0u;
    const uint32_t x = GRAIN ? (uint32_t)pix0 - y * (uint32_t)P.W : 0u;

    float v[NE];     // RGB order
    float nz[NE];
    union { word_t q[3]; T e[NE]; } u;
    if (VEC) {
      const word_t* src = reinterpret_cast<const word_t*>(in + e0);
      u.q[0] = __ldg(src); u.q[1] = __ldg(src + 1); u.q[2] = __ldg(src + 2);
    } else {
#pragma unroll
      for (int i = 0; i < NE; ++i) u.e[i] = in[e0 + i];
    }
#pragma unroll
    for (int j = 0; j < PX; ++j) {
#pragma unroll
      for (int c = 0; c < 3; ++c) v[3 * j + c] = Elem<T>::ld(u.e[3 * j + (BGR ? 2 - c : c)]);
    }
    if (has_ext) {   // external noise is [B,H,W,3] in RGB order (test path)
      const noise_t* ns = reinterpret_cast<const noise_t*>(P.ext_noise) + e0;
      if (VEC && sizeof(noise_t) == sizeof(T)) {
        union { word_t q[3]; noise_t e[NE]; } n;
        const word_t* nq = reinterpret_cast<const word_t*>(ns);
        n.q[0] = __ldg(nq); n.q[1] = __ldg(nq + 1); n.q[2] = __ldg(nq + 2);
#pragma unroll
        for (int i = 0; i < NE; ++i) nz[i] = noise_ld<noise_t>(n.e[i]);
      } else {
#pragma unroll
        for (int i = 0; i < NE; ++i) nz[i] = noise_ld<noise_t>(ns[i]);
      }
    }
    if (VEC) {
      // x is a multiple of PX (even): PX/2 whole generator pairs
#pragma unroll
      for (int j = 0; j < PX; j += 2) {
        float z[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (GRAIN) {
          if (has_ext) {
#pragma unroll
            for (int i = 0; i < 6; ++i) z[i] = nz[3 * j + i];
          } else {
            grain_pair_normals(grain_pair_bits(P.gkey, gf, (x >> 1) + (uint32_t)(j >> 1), y), z);
          }
        }
        process_pair<MASK, EXACT>(P, cmf, z, &v[3 * j]);
      }
    } else {
      float zr = 0.f, zg = 0.f, zb = 0.f;
      if (GRAIN) {
        if (has_ext) { zr = nz[0]; zg = nz[1]; zb = nz[2]; }
        else grain_pixel_normals(P.gkey, gf, x, y, zr, zg, zb);
      }
      process_pixel<MASK, EXACT>(P, cmf, zr, zg, zb, v[0], v[1], v[2]);
    }
#pragma unroll
    for (int j = 0; j < PX; ++j) {
#pragma unroll
      for (int c = 0; c < 3; ++c) u.e[3 * j + (BGR ? 2 - c : c)] = Elem<T>::st(v[3 * j + c]);
    }
    if (VEC) {
      word_t* dst = reinterpret_cast<word_t*>(out + e0);
      dst[0] = u.q[0]; dst[1] = u.q[1]; dst[2] = u.q[2];
    } else {
#pragma unroll
      for (int i = 0; i < NE; ++i) out[e0 + i] = u.e[i];
    }
  }
}

// LUT on 4-channel frames (alpha copied through): VRGDG_IV_Adjustments.py:341-343
template <typename T>
__global__ void __launch_bounds__(256)
k_lut_rgba(const T* __restrict__ in, T* __restrict__ out, int64_t npix, LutParams L) {
  for (int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x; p < npix; p += (int64_t)gridDim.x * 256) {
    const T* s = in + p * 4;
    float r = Elem<T>::ld(s[0]), g = Elem<T>::ld(s[1]), b = Elem<T>::ld(s[2]);
    T a = s[3];
    float x0 = r, x1 = g, x2 = b;
    lut3d_eval<true>(L, r, g, b);
    if (L.blend < 1.0f) {
      r = lut_blend<true>(x0, r, L.blend, L.one_minus_blend);
      g = lut_blend<true>(x1, g, L.blend, L.one_minus_blend);
      b = lut_blend<true>(x2, b, L.blend, L.one_minus_blend);
    }
    T* d = out + p * 4;
    d[0] = Elem<T>::st(r); d[1] = Elem<T>::st(g); d[2] = Elem<T>::st(b);
    d[3] = (L.blend < 1.0f) ? Elem<T>::st(lut_blend<true>(Elem<T>::ld(a), Elem<T>::ld(a), L.blend, L.one_minus_blend)) : a;
  }
}

// raw normals of the generator, [B,H,W,3] fp32
static __global__ void __launch_bounds__(256)
k_grain_noise(float* __restrict__ out, int B, int W, int64_t hw, uint64_t seed, int64_t frame0, int seed_mode, GrainKey K) {
  const int64_t total = (int64_t)B * hw;
  for (int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x; p < total; p += (int64_t)gridDim.x * 256) {
    int frame = (int)(p / hw);
    uint32_t pif = (uint32_t)(p - (int64_t)frame * hw);
    uint32_t y = pif / (uint32_t)W, x = pif - y * (uint32_t)W;
    GrainFrame gf = grain_frame(seed, frame0, frame, seed_mode);
    float zr, zg, zb;
    grain_pixel_normals(K, gf, x, y, zr, zg, zb);
    out[p * 3] = zr; out[p * 3 + 1] = zg; out[p * 3 + 2] = zb;
  }
}

// =====================================================================================================
// mbarrier / TMA primitives (inline PTX; SASS: SYNCS.*, UTMALDG)
// =====================================================================================================
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// Bounded wait: a lost TMA completion traps (reported as a CUDA error) instead of hanging the GPU.  The bound is WALL-CLOCK time
// (20 s on %globaltimer, far beyond any preemption by time-slicing / MPS / a debugger on a shared box), the spin backs off with
// nanosleep so that a long wait does not steal issue slots from the CTA that shares the SM.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
#pragma unroll 1
  for (int i = 0; i < 64; ++i)
    if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = globaltimer_ns();
  uint32_t ns = 32;
  while (!mbar_try_wait(bar, parity)) {
    __nanosleep(ns);
    if (ns < 1024) ns <<= 1;
    if (globaltimer_ns() - t0 > 20000000000ull) __trap();
  }
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* tmap, int c0, int c1, int c2,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(smem_u32(smem_dst)), "l"((uint64_t)tmap), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}

// =====================================================================================================
// k_tile — halo tiles staged in shared memory by TMA (3-stage mbarrier ring), optional per-pixel
// pre-stages applied to the whole halo tile in shared memory, 3x3 stencil, optional post grain.
// =====================================================================================================
struct TileParams {
  int B, H, W, RW;              // RW = 3*W elements per row
  int tiles_x, tiles_y;
  int64_t total_tiles;
  PointParams P;                // pre-stages
  int op;                       // VRGDG_STENCIL_*
  float strength;
  int border;                   // 0 replicate, 1 zero
  int post_enabled;
  float pI, ps, poms;
  uint64_t pseed;
  int64_t pframe0;
  int pseed_mode;
  GrainKey pkey;                // round keys of the post-grain generator
  int exact_stencil;            // 1: reference evaluation order, one rounding per op (bit-exact NumPy-path results for fp32)
  int use_tma;                  // 0: cooperative bounds-checked loads (any alignment)
  int vec_store;                // rows 16-byte aligned -> 16-byte stores
  int grid_limit;               // > 0: launch at most this many persistent CTAs (pipelined colour-match schedule leaves room for the statistics pass)
};

// HEAVY = the LUT gather runs in the pre-stage.  Two 256-thread CTAs per SM beat one 480-thread CTA on the fused grain + LUT + unsharp
// chain (while one CTA runs its stencil phase the other keeps the L1 gather busy); a third CTA runs out of registers, and 64-row tiles
// leave no room for a second CTA.  Two CTAs with a single staged
// tile each (the stage is refilled while the stencil runs, see EARLY in k_tile) leave ~120 KB of the SM's 228 KB as L1 for the table.
// Everything else uses 256-thread CTAs, a 3-stage ring and 2 CTAs per SM.
// WORK = 16-bit frames with pre-stages: their fp32 results live in a separate work tile, and a thread then produces
// 4 elements per row (16-byte shared loads at a 16-byte lane stride are bank-conflict free; 32-byte strides are not).
template <typename T, int MASK> struct TileCfg {
  static constexpr bool HEAVY = (MASK & ST_LUT) != 0;
  static constexpr bool WORK = (sizeof(T) == 1) || (((MASK & ST_PRE) != 0) && (sizeof(T) != 4));   // uint8 frames always convert into the work tile
  static constexpr bool GPLANE = (MASK & ST_POST) != 0;   // grain of the post stage, one Philox call per pixel pair, kept in its own fp32 plane
  static constexpr int VEC = WORK ? 4 : 16 / (int)sizeof(T);   // output elements per thread per row
  static constexpr int BX = 256;                      // box width (elements) = TMA inner-dimension limit
  static constexpr int PADL = 16 / (int)sizeof(T);    // box starts 16 BYTES left of the tile: TMA needs a 16-byte aligned start address
  static constexpr int TXE = sizeof(T) == 1 ? 192 : 240;   // output elements per tile row: multiple of 6 and of VEC, TXE*sizeof(T) % 16 == 0 (every box start
                                                            // must be 16-byte aligned: an unaligned start is an illegal instruction), PADL + TXE + 3 <= BX
#ifndef VRGDG_TILE_ROWS
#define VRGDG_TILE_ROWS 32
#endif
  static constexpr int TY = VRGDG_TILE_ROWS;          // output rows per tile
  static constexpr int ROWS = TY + 2;
#ifndef VRGDG_HEAVY_THREADS
#define VRGDG_HEAVY_THREADS 256
#endif
  static constexpr int THREADS = HEAVY ? VRGDG_HEAVY_THREADS : 256;
  // Register budget of the LUT configurations on fp32 frames: declaring a larger block than is ever launched lowers ptxas' register
  // cap (65536 / (LB_THREADS * MINB)) below the 128 that two 256-thread CTAs would allow, which leaves room in the register file for
  // the statistics blocks of the NEXT frame group next to two resident tile CTAs (pipelined colour-match schedule, vrgdg_abi.cu).
  // 256 (104-109 registers) fits one 128-thread statistics block beside two tile CTAs, 320 (91-94 registers) two, 352 (80 registers)
  // three or four.  At 80 registers the sm_90a LUT tile kernels spill 12-168 bytes per thread (ptxas -v).  352 was chosen by a sweep
  // on an earlier GPU with the same register file and shared memory per SM and has not been re-swept on H100.
#ifndef VRGDG_HEAVY_LB
#define VRGDG_HEAVY_LB 352
#endif
  static constexpr int LB_THREADS = (HEAVY && sizeof(T) == 4 && VRGDG_HEAVY_LB > THREADS) ? VRGDG_HEAVY_LB : THREADS;
#ifndef VRGDG_HEAVY_MINB
#define VRGDG_HEAVY_MINB 2
#endif
#ifndef VRGDG_HEAVY_NS
#define VRGDG_HEAVY_NS (WORK ? 1 : 2)                 // in-place (fp32) tiles need the staged tile until the stencil is done
#endif
#ifndef VRGDG_LIGHT_MINB
#define VRGDG_LIGHT_MINB 2
#endif
#ifndef VRGDG_LIGHT_NS
#define VRGDG_LIGHT_NS 3
#endif
  // plain stencils on 16-bit frames need few registers and 17 KB per staged tile: four CTAs per SM with a 2-stage ring
  // (fp32 tiles are 35 KB per stage and gain nothing from a third CTA)
  static constexpr bool SLIM = (MASK == 0) && (sizeof(T) == 2);
  static constexpr int MINB = HEAVY ? VRGDG_HEAVY_MINB : (SLIM ? 4 : VRGDG_LIGHT_MINB);
  static constexpr int COLS = TXE / VEC;              // threads across
  static constexpr int RG = (THREADS / COLS) >= 8 ? 8 : 4;   // row groups: COLS*RG active threads
  static constexpr int RPT = TY / RG;                 // rows per thread
  static constexpr int PPR = TXE / 3 + 2;             // halo-tile pixels per row
  static constexpr int PAIRS = PPR / 2 + 1;           // generator pixel pairs covering them (tile x origin is even)
  static constexpr int NS = HEAVY ? VRGDG_HEAVY_NS : ((GPLANE || SLIM) ? 2 : VRGDG_LIGHT_NS);   // pipeline stages
  static constexpr int STAGE_BYTES = ROWS * BX * (int)sizeof(T);
  static_assert(PADL + TXE + 3 <= BX, "box too narrow");
  static_assert(TY % RG == 0 && COLS * RG <= THREADS, "thread mapping");
};

template <typename T, int MASK>
constexpr size_t tile_smem_bytes() {
  using C = TileCfg<T, MASK>;
  size_t s = (size_t)C::NS * C::STAGE_BYTES;
  if (C::WORK) s += (size_t)C::ROWS * C::BX * 4;      // fp32 work tile
  if (C::GPLANE) s += (size_t)C::ROWS * C::BX * 4;    // post-grain plane
  return s + 64 /* mbarriers */ + 128 /* alignment slack */;
}

// replicate-border fix-up of a staged tile (np.pad(mode="edge") on the stage's input)
template <typename E, typename CFG>
__device__ __forceinline__ void fix_border(E* tile, int y0, int x0e, int H, int RW) {
  constexpr int BX = CFG::BX, ROWS = CFG::ROWS, PADL = CFG::PADL, TY = CFG::TY, TXE = CFG::TXE;
  const int vr = H - y0;        // image rows from y0 to the bottom
  const int ve = RW - x0e;      // row elements from x0e to the right edge
  const bool top = (y0 == 0), bot = (vr <= TY), left = (x0e == 0), right = (ve <= TXE);
  if (!(top || bot || left || right)) return;   // uniform per tile
  if (top || bot) {
    for (int c = threadIdx.x; c < BX; c += blockDim.x) {
      if (top) tile[c] = tile[BX + c];
      if (bot) tile[(vr + 1) * BX + c] = tile[vr * BX + c];
    }
  }
  __syncthreads();
  if (left || right) {
    for (int i = threadIdx.x; i < ROWS * 3; i += blockDim.x) {
      int r = i / 3, c = i - r * 3;
      E* row = tile + r * BX;
      if (left) row[PADL - 3 + c] = row[PADL + c];
      if (right) row[PADL + ve + c] = row[PADL + ve - 3 + c];
    }
  }
  __syncthreads();
}

// 128-bit shared load that the compiler cannot narrow: when only 3 of the 4 words are used it turns a plain float4 load into
// LDS.32 + LDS.64, and those run into 4-way bank conflicts at the 16-byte lane stride of the stencil (ncu: 35 % of the fused
// chain's shared wavefronts were excess).  Whole 16-byte accesses at a 16-byte lane stride are conflict free.
__device__ __forceinline__ uint4 lds128(const void* p) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(smem_u32(p)) : "memory");
  return v;
}

// window row: WN = VEC+6 floats starting at element (f0 - 3) of the tile row
template <typename E, int VEC>
__device__ __forceinline__ void load_window(const E* rowp /* -> tile column PADL+f0 */, float* w) {
  if (sizeof(E) == 4) {
    // floats [f0-4, f0+VEC+4): (VEC+8)/4 aligned 16-byte words
    constexpr int NV = (VEC + 8) / 4;
    float tmp[NV * 4];
    const float* p = reinterpret_cast<const float*>(rowp) - 4;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const uint4 q = lds128(p + 4 * i);
      tmp[4 * i] = __uint_as_float(q.x); tmp[4 * i + 1] = __uint_as_float(q.y);
      tmp[4 * i + 2] = __uint_as_float(q.z); tmp[4 * i + 3] = __uint_as_float(q.w);
    }
#pragma unroll
    for (int i = 0; i < VEC + 6; ++i) w[i] = tmp[i + 1];
  } else {
    // 16-bit elements [f0-8, f0+16): three aligned 16-byte words (VEC == 8)
    union { uint4 q[3]; E e[24]; } u;
    u.q[0] = lds128(rowp - 8); u.q[1] = lds128(rowp); u.q[2] = lds128(rowp + 8);
#pragma unroll
    for (int i = 0; i < VEC + 6; ++i) w[i] = Elem<E>::ld(u.e[i + 5]);
  }
}

// grain after the stencil (EnhancerNodes.py:285-293) on VEC consecutive row elements starting at element ge0
template <int VEC, bool BGR>
__device__ __forceinline__ void post_grain_elems(const TileParams& Q, const GrainFrame& gf, int ge0, int y, float* o) {
  const int pfirst = ge0 / 3, plast = (ge0 + VEC - 1) / 3;
  constexpr int NPR = (VEC + 1) / 3 + 1;                    // pixel pairs a run of VEC elements can touch
#pragma unroll
  for (int q = 0; q < NPR; ++q) {
    const int pair = (pfirst >> 1) + q;
    if (pair * 2 > plast) break;
    float z[6];
    grain_pair_normals(grain_pair_bits(Q.pkey, gf, (uint32_t)pair, (uint32_t)y), z);
    const float gy0 = Q.poms * z[1], gy1 = Q.poms * z[4];
    const float g0 = fmaf(2.0f * Q.ps, z[0], gy0), g1 = fmaf(Q.ps, z[1], gy0), g2 = fmaf(3.0f * Q.ps, z[2], gy0);
    const float g3 = fmaf(2.0f * Q.ps, z[3], gy1), g4 = fmaf(Q.ps, z[4], gy1), g5 = fmaf(3.0f * Q.ps, z[5], gy1);
#pragma unroll
    for (int e = 0; e < VEC; ++e) {
      const int idx = ge0 + e - pair * 6;                   // 0..5 inside this pair (memory order)
      if (idx >= 0 && idx < 6) {
        const float lo = (idx == 0) ? (BGR ? g2 : g0) : ((idx == 1) ? g1 : (BGR ? g0 : g2));
        const float hi = (idx == 3) ? (BGR ? g5 : g3) : ((idx == 4) ? g4 : (BGR ? g3 : g5));
        const float gv = (idx < 3) ? lo : hi;
        o[e] = clamp01(fmaf(Q.pI, gv, o[e]));
      }
    }
  }
}

template <typename T, int VEC>
__device__ __forceinline__ void store_elems(T* __restrict__ out, const TileParams& Q, int frame, int y, int ge0, const float* o) {
  if (y < Q.H && ge0 < Q.RW) {
    T* dst = out + ((int64_t)frame * Q.H + y) * Q.RW + ge0;
    if (Q.vec_store) {
      if (VEC * sizeof(T) == 16) {
        union { uint4 q; T e[VEC]; } u;
#pragma unroll
        for (int e = 0; e < VEC; ++e) u.e[e] = Elem<T>::st(o[e]);
        *reinterpret_cast<uint4*>(dst) = u.q;
      } else if (VEC * sizeof(T) == 8) {
        union { uint2 q; T e[VEC]; } u;
#pragma unroll
        for (int e = 0; e < VEC; ++e) u.e[e] = Elem<T>::st(o[e]);
        *reinterpret_cast<uint2*>(dst) = u.q;
      } else {
        union { uint32_t q; T e[VEC]; } u;
#pragma unroll
        for (int e = 0; e < VEC; ++e) u.e[e] = Elem<T>::st(o[e]);
        *reinterpret_cast<uint32_t*>(dst) = u.q;
      }
    } else {
#pragma unroll
      for (int e = 0; e < VEC; ++e) if (ge0 + e < Q.RW) dst[e] = Elem<T>::st(o[e]);
    }
  }
}

template <typename T, int OP, int MASK, bool XS>
__device__ __forceinline__ void stencil_rows(const T* raw, const float* work, const float* gplane, T* __restrict__ out,
                                             const TileParams& Q, int frame, int y0, int x0e) {
  using C = TileCfg<T, MASK>;
  constexpr bool WORK = C::WORK;
  constexpr int VEC = C::VEC, BX = C::BX, PADL = C::PADL, WN = VEC + 6;
  const int tid = threadIdx.x;
  if (tid >= C::COLS * C::RG) return;
  const int cx = tid % C::COLS, rg = tid / C::COLS;
  const int f0 = cx * VEC;
  const int ge0 = x0e + f0;                 // first output element in the row
  const int rbase = rg * C::RPT;            // first output row of this thread == smem row of its upper neighbour
  auto load_row = [&](int srow, float* dst) {
    if constexpr (WORK) load_window<float, VEC>(work + srow * BX + PADL + f0, dst);
    else load_window<T, VEC>(raw + srow * BX + PADL + f0, dst);
  };
  const GrainFrame pgf = grain_frame(Q.pseed, Q.pframe0, frame, Q.pseed_mode);
  if (OP == 1 && !XS) {
    // 3x3 box is separable: keep the horizontal 3-sums of the two previous rows (nodes.py:194-206)
    float h0[VEC], h1[VEC], c1[VEC], wr[WN];
    load_row(rbase, wr);
#pragma unroll
    for (int e = 0; e < VEC; ++e) h0[e] = (wr[e] + wr[e + 3]) + wr[e + 6];
    load_row(rbase + 1, wr);
#pragma unroll
    for (int e = 0; e < VEC; ++e) { h1[e] = (wr[e] + wr[e + 3]) + wr[e + 6]; c1[e] = wr[e + 3]; }
#pragma unroll
    for (int j = 0; j < C::RPT; ++j) {
      load_row(rbase + j + 2, wr);
      const int y = y0 + rbase + j;
      float o[VEC];
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        const float h2 = (wr[e] + wr[e + 3]) + wr[e + 6];
        const float blur = ((h0[e] + h1[e]) + h2) * 0.1111111111111111f;      // sum / 9.0 to within 1 ulp
        o[e] = clamp01(fmaf(Q.strength, c1[e] - blur, c1[e]));                 // img + s*(img - blur)
        h0[e] = h1[e]; h1[e] = h2; c1[e] = wr[e + 3];
      }
      if constexpr (C::GPLANE) {
        const float4* gp = reinterpret_cast<const float4*>(gplane + (rbase + j + 1) * BX + PADL + f0);
#pragma unroll
        for (int q = 0; q < VEC / 4; ++q) {
          const float4 gv = gp[q];
          o[4 * q] = clamp01(fmaf(Q.pI, gv.x, o[4 * q])); o[4 * q + 1] = clamp01(fmaf(Q.pI, gv.y, o[4 * q + 1]));
          o[4 * q + 2] = clamp01(fmaf(Q.pI, gv.z, o[4 * q + 2])); o[4 * q + 3] = clamp01(fmaf(Q.pI, gv.w, o[4 * q + 3]));
        }
      } else if ((MASK & ST_PRE) != 0 && Q.post_enabled) post_grain_elems<VEC, Io<T>::BGR>(Q, pgf, ge0, y, o);   // MASK 0 + post grain runs as ST_POST
      store_elems<T, VEC>(out, Q, frame, y, ge0, o);
    }
  } else {
    float w[3][WN];
    load_row(rbase, w[0]);
    load_row(rbase + 1, w[1]);
#pragma unroll
    for (int j = 0; j < C::RPT; ++j) {
      load_row(rbase + j + 2, w[2]);
      const int y = y0 + rbase + j;
      float o[VEC];
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        float n[9] = {w[0][e], w[0][e + 3], w[0][e + 6], w[1][e], w[1][e + 3], w[1][e + 6],
                      w[2][e], w[2][e + 3], w[2][e + 6]};
        o[e] = XS ? stencil_epilogue_exact(OP, n, Q.strength) : stencil_epilogue(OP, n, Q.strength);
      }
      if constexpr (C::GPLANE) {
        const float4* gp = reinterpret_cast<const float4*>(gplane + (rbase + j + 1) * BX + PADL + f0);
#pragma unroll
        for (int q = 0; q < VEC / 4; ++q) {
          const float4 gv = gp[q];
          o[4 * q] = clamp01(fmaf(Q.pI, gv.x, o[4 * q])); o[4 * q + 1] = clamp01(fmaf(Q.pI, gv.y, o[4 * q + 1]));
          o[4 * q + 2] = clamp01(fmaf(Q.pI, gv.z, o[4 * q + 2])); o[4 * q + 3] = clamp01(fmaf(Q.pI, gv.w, o[4 * q + 3]));
        }
      } else if ((MASK & ST_PRE) != 0 && Q.post_enabled) post_grain_elems<VEC, Io<T>::BGR>(Q, pgf, ge0, y, o);   // MASK 0 + post grain runs as ST_POST
      store_elems<T, VEC>(out, Q, frame, y, ge0, o);
#pragma unroll
      for (int i = 0; i < WN; ++i) { w[0][i] = w[1][i]; w[1][i] = w[2][i]; }
    }
  }
}

// six consecutive staged elements (even element offset) as three 2-element words
template <typename T>
__device__ __forceinline__ void pair_load6(const T* p, bool word0, float* e) {
  if (sizeof(T) == 4) {
    const float2* q = reinterpret_cast<const float2*>(p);
    if (word0) { float2 v = q[0]; e[0] = v.x; e[1] = v.y; }
    float2 v1 = q[1], v2 = q[2];
    e[2] = v1.x; e[3] = v1.y; e[4] = v2.x; e[5] = v2.y;
  } else if (sizeof(T) == 2) {
    const uint32_t* q = reinterpret_cast<const uint32_t*>(p);
    union { uint32_t u[3]; T h[6]; } w;
    w.u[0] = word0 ? q[0] : 0u; w.u[1] = q[1]; w.u[2] = q[2];
#pragma unroll
    for (int i = 0; i < 6; ++i) e[i] = Elem<T>::ld(w.h[i]);
  } else {
    const uint16_t* q = reinterpret_cast<const uint16_t*>(p);
    union { uint16_t u[3]; T h[6]; } w;
    w.u[0] = word0 ? q[0] : (uint16_t)0; w.u[1] = q[1]; w.u[2] = q[2];
#pragma unroll
    for (int i = 0; i < 6; ++i) e[i] = Elem<T>::ld(w.h[i]);
  }
}
__device__ __forceinline__ void pair_store6(float* p, bool word0, const float* e) {
  float2* q = reinterpret_cast<float2*>(p);
  if (word0) q[0] = make_float2(e[0], e[1]);
  q[1] = make_float2(e[2], e[3]);
  q[2] = make_float2(e[4], e[5]);
}

template <typename T, int MASK, bool EXACT>
__global__ void __launch_bounds__((TileCfg<T, MASK>::LB_THREADS), (TileCfg<T, MASK>::MINB))
k_tile(const __grid_constant__ CUtensorMap tmap, const T* __restrict__ in, T* __restrict__ out, TileParams Q) {
  using C = TileCfg<T, MASK>;
  constexpr int NT = C::THREADS;
  constexpr int VEC = C::VEC, BX = C::BX, PADL = C::PADL, TXE = C::TXE, TY = C::TY, ROWS = C::ROWS;
  constexpr int NS = C::NS;
  constexpr bool WORK = C::WORK;                           // separate fp32 tile for the pre-stage results

  extern __shared__ uint8_t smem_raw[];
  // 128-byte alignment by offset (keeps the pointer in the shared address space -> LDS/STS, not generic LD/ST)
  const uint32_t smem_a = smem_u32(smem_raw);
  uint8_t* base = smem_raw + (((smem_a + 127u) & ~127u) - smem_a);
  T* stage0 = reinterpret_cast<T*>(base);
  constexpr bool GPLANE = C::GPLANE;
  float* work = reinterpret_cast<float*>(base + (size_t)NS * C::STAGE_BYTES);
  float* gplane = reinterpret_cast<float*>(base + (size_t)NS * C::STAGE_BYTES + (WORK ? ROWS * BX * 4 : 0));
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + (size_t)NS * C::STAGE_BYTES + (WORK ? ROWS * BX * 4 : 0) + (GPLANE ? ROWS * BX * 4 : 0));

  const int tid = threadIdx.x;
  // total_tiles < 2^31 (checked on the host): 32-bit tile arithmetic, no 64-bit divisions per tile
  const uint32_t first = blockIdx.x, stride = gridDim.x, total = (uint32_t)Q.total_tiles;
  const uint32_t n_my = (total > first) ? (total - first + stride - 1) / stride : 0;
  const uint32_t tiles_per_frame = (uint32_t)(Q.tiles_x * Q.tiles_y);
  const bool tma = Q.use_tma != 0;

  if (tma && tid == 0) {
#pragma unroll
    for (int s = 0; s < NS; ++s) mbar_init(&bars[s], 1);
    fence_mbar_init();
    fence_proxy_async();
  }
  __syncthreads();

  auto tile_coords = [&](uint32_t k, int& frame, int& y0, int& x0e) {
    const uint32_t t = first + k * stride;
    const uint32_t f = t / tiles_per_frame;
    const uint32_t rem = t - f * tiles_per_frame;
    const uint32_t ty = rem / (uint32_t)Q.tiles_x;
    frame = (int)f;
    y0 = (int)ty * TY;
    x0e = (int)(rem - ty * (uint32_t)Q.tiles_x) * TXE;
  };
  auto issue = [&](uint32_t k) {
    int frame, y0, x0e;
    tile_coords(k, frame, y0, x0e);
    int s = (int)(k % NS);
    mbar_arrive_expect_tx(&bars[s], (uint32_t)C::STAGE_BYTES);
    tma_load_3d(reinterpret_cast<uint8_t*>(stage0) + (size_t)s * C::STAGE_BYTES, &tmap, x0e - PADL, y0 - 1, frame, &bars[s]);
  };

  // WORK configurations copy the staged tile into the fp32 work tile in the pre-stage, so the stage is free again as soon as
  // the pre-stage barrier has passed: its refill (tile k + NS) is issued there and overlaps the stencil phase; in-place
  // configurations refill at the top of the next iteration (tile k + NS - 1 into the stage the previous iteration used).
#ifndef VRGDG_EARLY_REFILL
#define VRGDG_EARLY_REFILL 1
#endif
  constexpr bool EARLY = WORK && (VRGDG_EARLY_REFILL != 0);
  // a single in-place stage (NS == 1 without a work tile) is refilled at the END of the iteration, once the stencil has read it;
  // the load latency is then covered by the other resident CTAs of the SM instead of a second stage
  constexpr bool LATE1 = !EARLY && NS == 1;
  constexpr uint32_t AHEAD = EARLY ? NS : (LATE1 ? 1 : NS - 1);
  if (tma && tid == 0) {
    for (uint32_t k = 0; k < AHEAD && k < n_my; ++k) issue(k);
  }

  for (uint32_t k = 0; k < n_my; ++k) {
    int frame, y0, x0e;
    tile_coords(k, frame, y0, x0e);
    const int s = tma ? (int)(k % NS) : 0;
    T* raw = reinterpret_cast<T*>(reinterpret_cast<uint8_t*>(stage0) + (size_t)s * C::STAGE_BYTES);

    if (tma) {
      if (!EARLY && !LATE1 && tid == 0 && k + NS - 1 < n_my) {
        fence_proxy_async();          // order earlier generic-proxy accesses of that stage before the async write
        issue(k + NS - 1);
      }
      mbar_wait(&bars[s], (uint32_t)((k / NS) & 1));
    } else {
      // generic loader: zero-filled halo tile, any alignment
      const T* fbase = in + (int64_t)frame * Q.H * Q.RW;
      for (int i = tid; i < ROWS * BX; i += NT) {
        int r = i / BX, c = i - r * BX;
        int y = y0 - 1 + r, x = x0e - PADL + c;
        T v = Elem<T>::st(0.0f);
        if (y >= 0 && y < Q.H && x >= 0 && x < Q.RW) v = fbase[(int64_t)y * Q.RW + x];
        raw[i] = v;
      }
      __syncthreads();
    }

    // ---- per-pixel pre-stages over the halo tile (grain / colour match / LUT), result in fp32 ----
    // one task = one generator pixel pair (2 horizontally adjacent pixels): one Philox call, two independent LUT gathers in flight
    if ((MASK & ST_PRE) != 0 || WORK || GPLANE) {
      const PointParams& P = Q.P;
      constexpr bool GRAIN = (MASK & ST_GRAIN) != 0;
      constexpr bool BGR = Io<T>::BGR;
      typedef typename Io<T>::noise_t noise_t;
      const GrainFrame gf = grain_frame(P.seed, P.frame0, frame, P.seed_mode);
      CmFold cmf = {};
      if (MASK & (ST_CM | ST_CMF)) cmf = cm_fold(P.cm_params + (int64_t)frame * 12, P.cm_t, P.cm_omt);
      const bool has_ext = GRAIN && (P.ext_noise != nullptr);
      const GrainFrame pgf = grain_frame(Q.pseed, Q.pframe0, frame, Q.pseed_mode);
      const int pair0 = x0e / 6 - 1;                        // pair holding the left halo pixel (x0e is a multiple of TXE, TXE of 6)
      for (int i = tid; i < ROWS * C::PAIRS; i += NT) {
        const int r = i / C::PAIRS, kx = i - r * C::PAIRS;
        const int y = y0 - 1 + r, pair = pair0 + kx;
        const int pxa = pair * 2;
        const int so = r * BX + PADL - 6 + 6 * kx;          // smem element of pixel a (outside the box for kx == 0)
        const bool rowin = (y >= 0 && y < Q.H);
        const bool need_a = (kx > 0), need_b = (kx < C::PAIRS - 1);
        const bool in_a = need_a && rowin && pxa >= 0 && pxa < Q.W;
        const bool in_b = need_b && rowin && pxa + 1 >= 0 && pxa + 1 < Q.W;
        // staged elements so..so+5 (pixel a = so..so+2, pixel b = so+3..so+5) move as three 2-element words: lane stride is
        // 6 elements, so 32/64-bit shared accesses are bank-conflict free.  Word 0 lies left of the box when kx == 0.
        if (GPLANE) {
          // post-grain values of this pair (added after the stencil): I*(s*z' + (1-s)*z_g) per element, memory channel order
          float gz[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          if (rowin && pair >= 0 && pxa < Q.W) {
            float z[6];
            grain_pair_normals(grain_pair_bits(Q.pkey, pgf, (uint32_t)pair, (uint32_t)y), z);
            const float gy0 = Q.poms * z[1], gy1 = Q.poms * z[4];
            const float r0 = fmaf(2.0f * Q.ps, z[0], gy0), g0 = fmaf(Q.ps, z[1], gy0), b0 = fmaf(3.0f * Q.ps, z[2], gy0);
            const float r1 = fmaf(2.0f * Q.ps, z[3], gy1), g1 = fmaf(Q.ps, z[4], gy1), b1 = fmaf(3.0f * Q.ps, z[5], gy1);
            gz[0] = BGR ? b0 : r0; gz[1] = g0; gz[2] = BGR ? r0 : b0;
            gz[3] = BGR ? b1 : r1; gz[4] = g1; gz[5] = BGR ? r1 : b1;
          }
          pair_store6(gplane + so, kx > 0, gz);
        }
        if ((MASK & ST_PRE) == 0 && !WORK) continue;               // nothing to do to the pixel values themselves
        float e[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (in_a | in_b) {
          pair_load6<T>(raw + so, kx > 0, e);
          float z[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          if (GRAIN) {
            if (has_ext) {
              const noise_t* ns = reinterpret_cast<const noise_t*>(P.ext_noise) + ((int64_t)frame * P.hw + (int64_t)y * Q.W + pxa) * 3;
              if (in_a) { z[0] = noise_ld<noise_t>(ns[0]); z[1] = noise_ld<noise_t>(ns[1]); z[2] = noise_ld<noise_t>(ns[2]); }
              if (in_b) { z[3] = noise_ld<noise_t>(ns[3]); z[4] = noise_ld<noise_t>(ns[4]); z[5] = noise_ld<noise_t>(ns[5]); }
            } else {
              grain_pair_normals(grain_pair_bits(P.gkey, gf, (uint32_t)pair, (uint32_t)y), z);
            }
          }
          // both pixels go through the stages unconditionally (their 2 x 3 LUT loads are then in flight together; a pixel
          // outside the image computes on staged zeros and is discarded) - the branchy form serialised the two gathers
          float p[6] = {e[BGR ? 2 : 0], e[1], e[BGR ? 0 : 2], e[BGR ? 5 : 3], e[4], e[BGR ? 3 : 5]};     // RGB for the stages
          process_pair<MASK, EXACT>(P, cmf, z, p);
          if (in_a) { e[BGR ? 2 : 0] = p[0]; e[1] = p[1]; e[BGR ? 0 : 2] = p[2]; } else if (WORK) { e[0] = 0.f; e[1] = 0.f; e[2] = 0.f; }
          if (in_b) { e[BGR ? 5 : 3] = p[3]; e[4] = p[4]; e[BGR ? 3 : 5] = p[5]; } else if (WORK) { e[3] = 0.f; e[4] = 0.f; e[5] = 0.f; }
        }
        if constexpr (WORK) {
          pair_store6(work + so, kx > 0, e);                       // zeros for pixels outside the image (memory channel order kept)
        } else {
          if (in_a | in_b) pair_store6(reinterpret_cast<float*>(raw) + so, kx > 0, e);   // in place; untouched pixels keep their staged value
        }
      }
      __syncthreads();
      if (EARLY && tma && tid == 0 && k + NS < n_my) {
        fence_proxy_async();          // the pre-stage's generic-proxy reads of this stage happen-before the async refill
        issue(k + NS);
      }
    }

    if (Q.border == 0) {
      if constexpr (WORK) fix_border<float, C>(work, y0, x0e, Q.H, Q.RW);
      else fix_border<T, C>(raw, y0, x0e, Q.H, Q.RW);
    }

    // ---- 3x3 stencil, sliding 3-row register window, VEC outputs per thread per row ----
    {
      const float* wt = WORK ? work : nullptr;
      if (Q.exact_stencil) {   // uniform; one specialised row loop per epilogue and arithmetic variant
        switch (Q.op) {
          case 1: stencil_rows<T, 1, MASK, true>(raw, wt, gplane, out, Q, frame, y0, x0e); break;
          case 2: stencil_rows<T, 2, MASK, true>(raw, wt, gplane, out, Q, frame, y0, x0e); break;
          case 3: stencil_rows<T, 3, MASK, false>(raw, wt, gplane, out, Q, frame, y0, x0e); break;
          case 4: stencil_rows<T, 4, MASK, true>(raw, wt, gplane, out, Q, frame, y0, x0e); break;
          case 5: stencil_rows<T, 5, MASK, false>(raw, wt, gplane, out, Q, frame, y0, x0e); break;
          default: stencil_rows<T, 0, MASK, false>(raw, wt, gplane, out, Q, frame, y0, x0e); break;
        }
      } else {
        switch (Q.op) {
          case 1: stencil_rows<T, 1, MASK, false>(raw, wt, gplane, out, Q, frame, y0, x0e); break;
          case 2: stencil_rows<T, 2, MASK, false>(raw, wt, gplane, out, Q, frame, y0, x0e); break;
          case 3: stencil_rows<T, 3, MASK, false>(raw, wt, gplane, out, Q, frame, y0, x0e); break;
          case 4: stencil_rows<T, 4, MASK, false>(raw, wt, gplane, out, Q, frame, y0, x0e); break;
          case 5: stencil_rows<T, 5, MASK, false>(raw, wt, gplane, out, Q, frame, y0, x0e); break;
          default: stencil_rows<T, 0, MASK, false>(raw, wt, gplane, out, Q, frame, y0, x0e); break;
        }
      }
    }
    if (tma) fence_proxy_async();   // generic-proxy writes to this stage happen-before its next async refill
    __syncthreads();   // every thread is done with this stage before it is refilled
    if (LATE1 && tma && tid == 0 && k + 1 < n_my) issue(k + 1);
  }
}

// =====================================================================================================
// LAB moments: per frame {S_L,S_a,S_b,S_LL,S_aa,S_bb} in fp64, fixed reduction order (deterministic).
// grid = (NB, B); each block writes one partial; k_moments_final folds the NB partials per frame.
// =====================================================================================================
// Partial sums per frame: 592 reduction units of 128 threads each, independent of B (results do not depend on sharding) and of the
// block size the kernel is launched with (a 256-thread block is two units), so every schedule produces bit-identical statistics.
constexpr int MOMENT_BLOCKS = 592;
constexpr int MOMENT_UNIT = 128;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// u = (fy, fx - fy, fy - fz) of one pixel (Lab is an affine image of u, see cm_sums_to_lab_host); (r, g, b) <- (fx, fy, fz)
__device__ __forceinline__ void moments_add(float& r, float& g, float& b, float* s1, float* s2) {
  float fx, fy, fz;
  rgb_to_fxyz(r, g, b, fx, fy, fz);
  r = fx; g = fy; b = fz;
  const float u1 = fx - fy, u2 = fy - fz;
  s1[0] += fy; s1[1] += u1; s1[2] += u2;
  s2[0] = fmaf(fy, fy, s2[0]); s2[1] = fmaf(u1, u1, s2[1]); s2[2] = fmaf(u2, u2, s2[2]);
}

// VEC: a thread moves 3 machine words = PX whole pixels per iteration (like k_point), one Philox call per pixel pair, the PX
// pixels' sums are formed in fp32 (<= 8 terms) and then added to the thread's fp64 accumulators.  !VEC: one pixel per iteration.
// fplanes != null (fp32 frames, VEC): the pass also stores (fx, fy, fz) of every pixel, [B][H][W][3] fp32 like the frames, for the
// ST_CMF second pass.
// NT = 256 (two reduction units per block) or 128 (one: small enough to share an SM with two resident tile CTAs, see
// vrgdg_chain_cm_apply's pipelined schedule).
#ifndef VRGDG_MOMENT_SMALL_MINB
#define VRGDG_MOMENT_SMALL_MINB 10     // 128-thread blocks per SM the register cap is computed for: 8 = 64 registers (three blocks fit beside two
                                       // 80-register tile CTAs), 10 = 48 registers (four blocks; no spills on sm_90a; chosen on an earlier GPU, not re-swept on H100)
#endif
template <int NT> struct MomentLaunch { static constexpr int MINB = (NT == MOMENT_UNIT) ? VRGDG_MOMENT_SMALL_MINB : 4; };   // 256 threads: 64 registers as before
template <typename T, bool GRAIN, bool VEC, int NT>
__global__ void __launch_bounds__(NT, (MomentLaunch<NT>::MINB))
k_lab_moments(const T* __restrict__ in, PointParams P, int row0, int rows, double* __restrict__ partials, float* __restrict__ fplanes) {
  static_assert(NT % MOMENT_UNIT == 0, "whole reduction units per block");
  constexpr int UPB = NT / MOMENT_UNIT;                       // units per block
  const int unit = blockIdx.x * UPB + (threadIdx.x / MOMENT_UNIT), ut = threadIdx.x % MOMENT_UNIT;
  typedef typename Io<T>::word_t word_t;
  typedef typename Io<T>::noise_t noise_t;
  constexpr bool BGR = Io<T>::BGR;
  constexpr int PX = VEC ? (int)(sizeof(word_t) / sizeof(T)) : 1;
  constexpr int NE = PX * 3;
  const int frame = blockIdx.y;
  const int64_t pbeg = (int64_t)row0 * P.W, n = (int64_t)rows * P.W;
  const T* fbase = in + (int64_t)frame * P.hw * 3;
  const GrainFrame gf = grain_frame(P.seed, P.frame0, frame, P.seed_mode);
  const bool has_ext = GRAIN && (P.ext_noise != nullptr);
  const CmFold nocm = {};
  double acc[6] = {0, 0, 0, 0, 0, 0};
  const int64_t groups = (n + PX - 1) / PX;      // VEC: n % PX == 0 (host-checked)
  for (int64_t gi = (int64_t)unit * MOMENT_UNIT + ut; gi < groups; gi += (int64_t)MOMENT_BLOCKS * MOMENT_UNIT) {
    const int64_t pif = pbeg + gi * PX;
    float v[NE], nz[NE];
    union { word_t q[3]; T e[NE]; } u;
    if (VEC) {
      const word_t* src = reinterpret_cast<const word_t*>(fbase + pif * 3);
      u.q[0] = __ldg(src); u.q[1] = __ldg(src + 1); u.q[2] = __ldg(src + 2);
    } else {
#pragma unroll
      for (int i = 0; i < NE; ++i) u.e[i] = fbase[pif * 3 + i];
    }
#pragma unroll
    for (int j = 0; j < PX; ++j) {
#pragma unroll
      for (int c = 0; c < 3; ++c) v[3 * j + c] = Elem<T>::ld(u.e[3 * j + (BGR ? 2 - c : c)]);
    }
    if (GRAIN) {
      const uint32_t y = (uint32_t)pif / (uint32_t)P.W, x = (uint32_t)pif - y * (uint32_t)P.W;
      if (has_ext) {
        const noise_t* ns = reinterpret_cast<const noise_t*>(P.ext_noise) + ((int64_t)frame * P.hw + pif) * 3;
#pragma unroll
        for (int i = 0; i < NE; ++i) nz[i] = noise_ld<noise_t>(ns[i]);
#pragma unroll
        for (int j = 0; j < PX; ++j)
          process_pixel<ST_GRAIN, true>(P, nocm, nz[3 * j], nz[3 * j + 1], nz[3 * j + 2], v[3 * j], v[3 * j + 1], v[3 * j + 2]);
      } else if (VEC) {
#pragma unroll
        for (int j = 0; j < PX; j += 2) {          // x is a multiple of PX (even): whole generator pairs
          float z[6];
          grain_pair_normals(grain_pair_bits(P.gkey, gf, (x >> 1) + (uint32_t)(j >> 1), y), z);
          process_pixel<ST_GRAIN, false>(P, nocm, z[0], z[1], z[2], v[3 * j], v[3 * j + 1], v[3 * j + 2]);
          process_pixel<ST_GRAIN, false>(P, nocm, z[3], z[4], z[5], v[3 * j + 3], v[3 * j + 4], v[3 * j + 5]);
        }
      } else {
        float zr, zg, zb;
        grain_pixel_normals(P.gkey, gf, x, y, zr, zg, zb);
        process_pixel<ST_GRAIN, false>(P, nocm, zr, zg, zb, v[0], v[1], v[2]);
      }
    }
    float s1[3] = {0.f, 0.f, 0.f}, s2[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < PX; ++j) moments_add(v[3 * j], v[3 * j + 1], v[3 * j + 2], s1, s2);
#pragma unroll
    for (int c = 0; c < 3; ++c) { acc[c] += (double)s1[c]; acc[3 + c] += (double)s2[c]; }
    if constexpr (VEC && sizeof(T) == 4) {
      if (fplanes != nullptr) {                  // uniform; v now holds (fx, fy, fz) per pixel
        float4* dst = reinterpret_cast<float4*>(fplanes + ((int64_t)frame * P.hw + pif) * 3);
        dst[0] = make_float4(v[0], v[1], v[2], v[3]);
        dst[1] = make_float4(v[4], v[5], v[6], v[7]);
        dst[2] = make_float4(v[8], v[9], v[10], v[11]);
      }
    }
  }
  __shared__ double red[NT / 32][6];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < 6; ++q) {
    double v = warp_sum(acc[q]);
    if (lane == 0) red[wid][q] = v;
  }
  __syncthreads();
  if (ut < 6) {                                               // one partial per 128-thread unit: its four warps in order
    const int w0 = (threadIdx.x / MOMENT_UNIT) * (MOMENT_UNIT / 32);
    double v = 0;
#pragma unroll
    for (int w = 0; w < MOMENT_UNIT / 32; ++w) v += red[w0 + w][ut];
    partials[((int64_t)frame * MOMENT_BLOCKS + unit) * 6 + ut] = v;
  }
}

// sums[frame] = {n, S_L, S_a, S_b, S_LL, S_aa, S_bb}: fold of the block partials (sums over u = (fy, fx-fy, fy-fz)) in a fixed
// order, then the affine change of variables u -> Lab in fp64 (cm_sums_to_lab_host)
static __global__ void k_moments_final(const double* __restrict__ partials, int nb, double n, double* __restrict__ sums) {
  const int frame = blockIdx.x, lane = threadIdx.x;   // 32 threads
  double acc[6] = {0, 0, 0, 0, 0, 0};
  for (int b = lane; b < nb; b += 32) {
#pragma unroll
    for (int q = 0; q < 6; ++q) acc[q] += partials[((int64_t)frame * nb + b) * 6 + q];
  }
#pragma unroll
  for (int q = 0; q < 6; ++q) acc[q] = warp_sum(acc[q]);
  if (lane == 0) {
    double* o = sums + (int64_t)frame * 7;
    o[0] = n;
    o[1] = 116.0 * acc[0] - 16.0 * n;
    o[2] = 500.0 * acc[1];
    o[3] = 200.0 * acc[2];
    o[4] = 13456.0 * acc[3] - 3712.0 * acc[0] + 256.0 * n;
    o[5] = 250000.0 * acc[4];
    o[6] = 40000.0 * acc[5];
  }
}

// params[b] = {k[3] = sd_ref/sd_img, c0[3] = mu_ref - mu_img*k, mu_img[3], sd_img[3]};  sd = sqrt(unbiased var) + 1e-5
// (nodes.py:99-100,109-110); k and c0 are formed in fp64 and rounded once, so that matched = lab*k + c0 (one FMA)
static __global__ void k_colormatch_params(const double* __restrict__ fs, int B, const double* __restrict__ rs, int n_ref,
                                    float* __restrict__ params) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const double* f = fs + (int64_t)b * 7;
  const double* r = rs + (int64_t)((n_ref == 1) ? 0 : b) * 7;
  float* p = params + (int64_t)b * 12;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    double n = f[0], m = f[1 + c] / n;
    double var = (f[4 + c] - f[1 + c] * m) / (n - 1.0);
    const float sd = __fadd_rn((float)sqrt(var > 0 ? var : 0.0), 1e-5f);        // fp32 std + 1e-5 as the reference forms it
    double nr = r[0], mr = r[1 + c] / nr;
    double varr = (r[4 + c] - r[1 + c] * mr) / (nr - 1.0);
    const float sdr = __fadd_rn((float)sqrt(varr > 0 ? varr : 0.0), 1e-5f);
    const double k = (double)sdr / (double)sd;
    p[c] = (float)k;
    p[3 + c] = (float)((double)(float)mr - (double)(float)m * k);               // the reference's means are fp32 tensors
    p[6 + c] = (float)m;
    p[9 + c] = sd;
  }
}

// reference-layout table [S][S][S][3] -> cell table (see vrgdg_math.cuh)
static __global__ void __launch_bounds__(256)
k_lut_pack(const float* __restrict__ lut3, float* __restrict__ cells, int S) {
  const int n = S * S * S;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
    const int r = i % S, g = (i / S) % S, b = i / (S * S);
    float e[LUT_CELL_FLOATS];
    lut_pack_entry(lut3, S, b, g, r, e);
    float4* d = reinterpret_cast<float4*>(cells + (size_t)i * LUT_CELL_FLOATS);
#pragma unroll
    for (int k = 0; k < LUT_CELL_FLOATS / 4; ++k) d[k] = make_float4(e[4 * k], e[4 * k + 1], e[4 * k + 2], e[4 * k + 3]);
  }
}

// polynomial cell table of the fast chains (vrgdg_math.cuh "polynomial cells")
static __global__ void __launch_bounds__(256)
k_lutp_pack(const float* __restrict__ lut3, float* __restrict__ cells, int S) {
  const int n = S * S * S;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
    const int r = i % S, g = (i / S) % S, b = i / (S * S);
    float e[LUT_CELL_FLOATS];
    lutp_pack_entry(lut3, S, b, g, r, e);
    float4* d = reinterpret_cast<float4*>(cells + (size_t)i * LUT_CELL_FLOATS);
#pragma unroll
    for (int k = 0; k < LUT_CELL_FLOATS / 4; ++k) d[k] = make_float4(e[4 * k], e[4 * k + 1], e[4 * k + 2], e[4 * k + 3]);
  }
}

// =====================================================================================================
// uint8 BGR wire format (VRGDG_LUTVideoTools.py:736-752): 4 pixels (12 bytes) per thread
// =====================================================================================================
template <typename T>
__global__ void __launch_bounds__(256)
k_u8bgr_to_rgb(const uint8_t* __restrict__ in, T* __restrict__ out, int64_t npix) {
  for (int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x; p < npix; p += (int64_t)gridDim.x * 256) {
    const uint8_t* s = in + p * 3;
    float b = (float)s[0], g = (float)s[1], r = (float)s[2];
    T* d = out + p * 3;
    d[0] = Elem<T>::st(divx(r, 255.0f));     // astype(float32) / 255.0
    d[1] = Elem<T>::st(divx(g, 255.0f));
    d[2] = Elem<T>::st(divx(b, 255.0f));
  }
}
template <typename T>
__global__ void __launch_bounds__(256)
k_rgb_to_u8bgr(const T* __restrict__ in, uint8_t* __restrict__ out, int64_t npix) {
  for (int64_t p = (int64_t)blockIdx.x * 256 + threadIdx.x; p < npix; p += (int64_t)gridDim.x * 256) {
    const T* s = in + p * 3;
    float r = Elem<T>::ld(s[0]), g = Elem<T>::ld(s[1]), b = Elem<T>::ld(s[2]);
    // np.clip(x * 255.0, 0, 255).astype(uint8): truncation
    uint8_t* d = out + p * 3;
    d[0] = (uint8_t)fminf(fmaxf(mulx(b, 255.0f), 0.0f), 255.0f);
    d[1] = (uint8_t)fminf(fmaxf(mulx(g, 255.0f), 0.0f), 255.0f);
    d[2] = (uint8_t)fminf(fmaxf(mulx(r, 255.0f), 0.0f), 255.0f);
  }
}

// ---- host-side launchers implemented per dtype translation unit (vrgdg_inst.cuh) --------------------
struct LaunchCtx { cudaStream_t stream; int sms; };

template <typename T> cudaError_t launch_point(const void* in, void* out, const PointParams& P, int mask, bool exact,
                                               const LaunchCtx& ctx);
template <typename T> cudaError_t launch_lut_rgba(const void* in, void* out, int64_t npix, const LutParams& L,
                                                  const LaunchCtx& ctx);
template <typename T> cudaError_t launch_tile(const CUtensorMap* tmap, const void* in, void* out, TileParams& Q, int mask,
                                              bool exact, const LaunchCtx& ctx);
template <typename T> cudaError_t launch_moments(const void* in, const PointParams& P, bool grain, int row0, int rows,
                                                 double* sums, double* partials, const LaunchCtx& ctx, float* fplanes = nullptr,
                                                 bool small_blocks = false);
template <typename T> cudaError_t launch_u8_in(const uint8_t* in, void* out, int64_t npix, const LaunchCtx& ctx);
template <typename T> cudaError_t launch_u8_out(const void* in, uint8_t* out, int64_t npix, const LaunchCtx& ctx);
template <typename T> void tile_geometry(int H, int RW, int& tiles_x, int& tiles_y, int& box_x, int& box_y);

void count_launch();

}  // namespace vrgdg

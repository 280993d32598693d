// tools/lut_bench.cu — exploration micro-benchmark for the 3D-LUT gather (not part of the product).
// Build:  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o tools/lut_bench.bin tools/lut_bench.cu
// Compares table layouts / load widths / smem residency on white and natural-like frames.
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdio.h>
#include <stdint.h>
#include <stdlib.h>
#include <math.h>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

template <bool EXACT> __device__ __forceinline__ float lerp1(float a, float b, float f, float omf) {
  if (EXACT) return __fadd_rn(__fmul_rn(a, omf), __fmul_rn(b, f));
  return fmaf(f, b - a, a);
}

struct Idx { int r0, r1, g0, g1, b0, b1; float fr, fg, fb; };

template <bool DIV> __device__ __forceinline__ void coord(float v, float smax, int S, int& i0, int& i1, float& f) {
  float n = DIV ? __fdiv_rn(__fsub_rn(v, 0.0f), 1.0f + 0.0f * v) : v;   // DIV variant keeps a real division in the code
  n = clamp01(n);
  float c = __fmul_rn(n, smax);
  float fl = floorf(c);
  i0 = (int)fl; i1 = min(i0 + 1, S - 1); f = c - fl;
}

// ---- variant A/B: [S^3][3] scalar loads --------------------------------------------------------
#define LDV(p) (SMEM ? *(p) : __ldg(p))
template <bool EXACT, bool DIV, bool SMEM = false>
__device__ __forceinline__ void eval_scalar(const float* __restrict__ L, int S, float& r, float& g, float& b) {
  Idx q; float smax = (float)(S - 1);
  coord<DIV>(r, smax, S, q.r0, q.r1, q.fr); coord<DIV>(g, smax, S, q.g0, q.g1, q.fg); coord<DIV>(b, smax, S, q.b0, q.b1, q.fb);
  const float* p000 = L + ((q.b0 * S + q.g0) * S + q.r0) * 3; const float* p001 = L + ((q.b1 * S + q.g0) * S + q.r0) * 3;
  const float* p010 = L + ((q.b0 * S + q.g1) * S + q.r0) * 3; const float* p011 = L + ((q.b1 * S + q.g1) * S + q.r0) * 3;
  const float* p100 = L + ((q.b0 * S + q.g0) * S + q.r1) * 3; const float* p101 = L + ((q.b1 * S + q.g0) * S + q.r1) * 3;
  const float* p110 = L + ((q.b0 * S + q.g1) * S + q.r1) * 3; const float* p111 = L + ((q.b1 * S + q.g1) * S + q.r1) * 3;
  float omb = 1.f - q.fb, omg = 1.f - q.fg, omr = 1.f - q.fr, o[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float c00 = lerp1<EXACT>(LDV(p000 + c), LDV(p001 + c), q.fb, omb), c01 = lerp1<EXACT>(LDV(p010 + c), LDV(p011 + c), q.fb, omb);
    float c10 = lerp1<EXACT>(LDV(p100 + c), LDV(p101 + c), q.fb, omb), c11 = lerp1<EXACT>(LDV(p110 + c), LDV(p111 + c), q.fb, omb);
    o[c] = clamp01(lerp1<EXACT>(lerp1<EXACT>(c00, c01, q.fg, omg), lerp1<EXACT>(c10, c11, q.fg, omg), q.fr, omr));
  }
  r = o[0]; g = o[1]; b = o[2];
}

// ---- variant C: float4-packed [S^3] ----------------------------------------------------------------
template <bool EXACT, typename LD>
__device__ __forceinline__ void eval_f4(LD ld, int S, float& r, float& g, float& b) {
  Idx q; float smax = (float)(S - 1);
  coord<false>(r, smax, S, q.r0, q.r1, q.fr); coord<false>(g, smax, S, q.g0, q.g1, q.fg); coord<false>(b, smax, S, q.b0, q.b1, q.fb);
  float4 v000 = ld((q.b0 * S + q.g0) * S + q.r0), v001 = ld((q.b1 * S + q.g0) * S + q.r0);
  float4 v010 = ld((q.b0 * S + q.g1) * S + q.r0), v011 = ld((q.b1 * S + q.g1) * S + q.r0);
  float4 v100 = ld((q.b0 * S + q.g0) * S + q.r1), v101 = ld((q.b1 * S + q.g0) * S + q.r1);
  float4 v110 = ld((q.b0 * S + q.g1) * S + q.r1), v111 = ld((q.b1 * S + q.g1) * S + q.r1);
  float omb = 1.f - q.fb, omg = 1.f - q.fg, omr = 1.f - q.fr;
#define CH(m) clamp01(lerp1<EXACT>(lerp1<EXACT>(lerp1<EXACT>(v000.m, v001.m, q.fb, omb), lerp1<EXACT>(v010.m, v011.m, q.fb, omb), q.fg, omg), \
                                   lerp1<EXACT>(lerp1<EXACT>(v100.m, v101.m, q.fb, omb), lerp1<EXACT>(v110.m, v111.m, q.fb, omb), q.fg, omg), q.fr, omr))
  float o0 = CH(x), o1 = CH(y), o2 = CH(z);
#undef CH
  r = o0; g = o1; b = o2;
}

// ---- variant D/E: pair-packed [S^2*S] x {rgb(r0), pad, rgb(r0+1), pad} = 32 B ------------------------------
struct F8 { float4 a, b; };
__device__ __forceinline__ F8 ld256(const float* p) {
  F8 v;
  // sm_90 has no 256-bit load: one 32-byte sector as two 128-bit non-coherent loads
  asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.a.x), "=f"(v.a.y), "=f"(v.a.z), "=f"(v.a.w) : "l"(p));
  asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4+16];" : "=f"(v.b.x), "=f"(v.b.y), "=f"(v.b.z), "=f"(v.b.w) : "l"(p));
  return v;
}
__device__ __forceinline__ F8 ld2x128(const float* p) {
  F8 v; v.a = __ldg(reinterpret_cast<const float4*>(p)); v.b = __ldg(reinterpret_cast<const float4*>(p) + 1); return v;
}
template <bool EXACT, bool WIDE>
__device__ __forceinline__ void eval_pair(const float* __restrict__ P, int S, float& r, float& g, float& b) {
  Idx q; float smax = (float)(S - 1);
  coord<false>(r, smax, S, q.r0, q.r1, q.fr); coord<false>(g, smax, S, q.g0, q.g1, q.fg); coord<false>(b, smax, S, q.b0, q.b1, q.fb);
  auto L = [&](int bi, int gi) { const float* p = P + (size_t)(((bi * S + gi) * S + q.r0)) * 8; return WIDE ? ld256(p) : ld2x128(p); };
  F8 v00 = L(q.b0, q.g0), v01 = L(q.b1, q.g0), v10 = L(q.b0, q.g1), v11 = L(q.b1, q.g1);
  float omb = 1.f - q.fb, omg = 1.f - q.fg, omr = 1.f - q.fr;
#define CH(m) clamp01(lerp1<EXACT>(lerp1<EXACT>(lerp1<EXACT>(v00.a.m, v01.a.m, q.fb, omb), lerp1<EXACT>(v10.a.m, v11.a.m, q.fb, omb), q.fg, omg), \
                                   lerp1<EXACT>(lerp1<EXACT>(v00.b.m, v01.b.m, q.fb, omb), lerp1<EXACT>(v10.b.m, v11.b.m, q.fb, omb), q.fg, omg), q.fr, omr))
  float o0 = CH(x), o1 = CH(y), o2 = CH(z);
#undef CH
  r = o0; g = o1; b = o2;
}

// ---- variant 10: cell-packed [S^3] x 24 floats (8 corners x rgb) = 96 B, three 256-bit loads ----------------
template <bool EXACT>
__device__ __forceinline__ void eval_cell(const float* __restrict__ C, int S, float& r, float& g, float& b) {
  Idx q; float smax = (float)(S - 1);
  coord<false>(r, smax, S, q.r0, q.r1, q.fr); coord<false>(g, smax, S, q.g0, q.g1, q.fg); coord<false>(b, smax, S, q.b0, q.b1, q.fb);
  const float* p = C + (size_t)((q.b0 * S + q.g0) * S + q.r0) * 24;
  F8 a = ld256(p), c = ld256(p + 8), d = ld256(p + 16);
  // order: c000 c100 c010 c110 c001 c101 c011 c111, 3 floats each
  float v[24] = {a.a.x, a.a.y, a.a.z, a.a.w, a.b.x, a.b.y, a.b.z, a.b.w, c.a.x, c.a.y, c.a.z, c.a.w, c.b.x, c.b.y, c.b.z, c.b.w,
                 d.a.x, d.a.y, d.a.z, d.a.w, d.b.x, d.b.y, d.b.z, d.b.w};
  float omb = 1.f - q.fb, omg = 1.f - q.fg, omr = 1.f - q.fr, o[3];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    float c00 = lerp1<EXACT>(v[0 + ch], v[12 + ch], q.fb, omb), c10 = lerp1<EXACT>(v[3 + ch], v[15 + ch], q.fb, omb);
    float c01 = lerp1<EXACT>(v[6 + ch], v[18 + ch], q.fb, omb), c11 = lerp1<EXACT>(v[9 + ch], v[21 + ch], q.fb, omb);
    o[ch] = clamp01(lerp1<EXACT>(lerp1<EXACT>(c00, c01, q.fg, omg), lerp1<EXACT>(c10, c11, q.fg, omg), q.fr, omr));
  }
  r = o[0]; g = o[1]; b = o[2];
}

// ---- variant 11: cell-packed unorm21: 8 corners x 8 B = 64 B, two 256-bit loads; values must lie in [0,1] --------
__device__ __forceinline__ void dec21(uint32_t w0, uint32_t w1, float& r, float& g, float& b) {
  const uint32_t M = 0x1FFFFFu, C = 0x4B000000u;                  // float(k) = as_float(C | k) - 2^23 for k < 2^23
  r = __uint_as_float((w0 & M) | C) - 8388608.0f;
  g = __uint_as_float((__funnelshift_r(w0, w1, 21) & M) | C) - 8388608.0f;
  b = __uint_as_float(((w1 >> 10) & M) | C) - 8388608.0f;
}
__device__ __forceinline__ void eval_cell21(const float* __restrict__ Cq, int S, float& r, float& g, float& b) {
  Idx q; float smax = (float)(S - 1);
  coord<false>(r, smax, S, q.r0, q.r1, q.fr); coord<false>(g, smax, S, q.g0, q.g1, q.fg); coord<false>(b, smax, S, q.b0, q.b1, q.fb);
  const float* p = Cq + (size_t)((q.b0 * S + q.g0) * S + q.r0) * 16;
  F8 lo = ld256(p), hi = ld256(p + 8);
  uint32_t w[16] = {__float_as_uint(lo.a.x), __float_as_uint(lo.a.y), __float_as_uint(lo.a.z), __float_as_uint(lo.a.w),
                    __float_as_uint(lo.b.x), __float_as_uint(lo.b.y), __float_as_uint(lo.b.z), __float_as_uint(lo.b.w),
                    __float_as_uint(hi.a.x), __float_as_uint(hi.a.y), __float_as_uint(hi.a.z), __float_as_uint(hi.a.w),
                    __float_as_uint(hi.b.x), __float_as_uint(hi.b.y), __float_as_uint(hi.b.z), __float_as_uint(hi.b.w)};
  float v[8][3];
#pragma unroll
  for (int k = 0; k < 8; ++k) dec21(w[2 * k], w[2 * k + 1], v[k][0], v[k][1], v[k][2]);
  float o[3];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {       // corner order c000 c100 c010 c110 | c001 c101 c011 c111 (x=r, y=g, z=b)
    float c00 = fmaf(q.fb, v[4][ch] - v[0][ch], v[0][ch]), c10 = fmaf(q.fb, v[5][ch] - v[1][ch], v[1][ch]);
    float c01 = fmaf(q.fb, v[6][ch] - v[2][ch], v[2][ch]), c11 = fmaf(q.fb, v[7][ch] - v[3][ch], v[3][ch]);
    float c0 = fmaf(q.fg, c01 - c00, c00), c1 = fmaf(q.fg, c11 - c10, c10);
    o[ch] = clamp01(fmaf(q.fr, c1 - c0, c0) * 4.76837158203125e-07f);
  }
  r = o[0]; g = o[1]; b = o[2];
}

template <typename T> struct E;
template <> struct E<float> { static __device__ float ld(float v) { return v; } static __device__ float st(float v) { return v; } };
template <> struct E<__half> { static __device__ float ld(__half v) { return __half2float(v); } static __device__ __half st(float v) { return __float2half_rn(v); } };

// VAR: 0 scalar exact+div, 1 scalar exact, 2 f4 exact, 3 f4 fast, 4 pair 2x128 exact, 5 pair 256 exact, 6 pair 256 fast,
//      7 smem scalar [S^3][3] exact, 8 smem f4 exact, 9 passthrough (I/O only)
template <typename T, int VAR>
__global__ void __launch_bounds__(256) k_lut(const T* __restrict__ in, T* __restrict__ out, int64_t npix, const float* __restrict__ lut3,
                                              const float4* __restrict__ lut4, const float* __restrict__ lutp, int S,
                                              const float* __restrict__ lutc = nullptr, const float* __restrict__ lutq = nullptr) {
  extern __shared__ float4 sm4[];
  float* sm = reinterpret_cast<float*>(sm4);
  if (VAR == 7) { for (int i = threadIdx.x; i < S * S * S * 3; i += 256) sm[i] = lut3[i]; __syncthreads(); }
  if (VAR == 8) { for (int i = threadIdx.x; i < S * S * S; i += 256) sm4[i] = lut4[i]; __syncthreads(); }
  constexpr int PX = 48 / (3 * sizeof(T));
  const int64_t ngroups = npix / PX;
  for (int64_t grp = (int64_t)blockIdx.x * 256 + threadIdx.x; grp < ngroups; grp += (int64_t)gridDim.x * 256) {
    union { uint4 q[3]; T e[PX * 3]; } u;
    const uint4* src = reinterpret_cast<const uint4*>(in + grp * PX * 3);
    u.q[0] = __ldg(src); u.q[1] = __ldg(src + 1); u.q[2] = __ldg(src + 2);
#pragma unroll
    for (int j = 0; j < PX; ++j) {
      float r = E<T>::ld(u.e[3 * j]), g = E<T>::ld(u.e[3 * j + 1]), b = E<T>::ld(u.e[3 * j + 2]);
      if (VAR == 0) eval_scalar<true, true>(lut3, S, r, g, b);
      if (VAR == 1) eval_scalar<true, false>(lut3, S, r, g, b);
      if (VAR == 2) eval_f4<true>([&](int i) { return __ldg(lut4 + i); }, S, r, g, b);
      if (VAR == 3) eval_f4<false>([&](int i) { return __ldg(lut4 + i); }, S, r, g, b);
      if (VAR == 4) eval_pair<true, false>(lutp, S, r, g, b);
      if (VAR == 5) eval_pair<true, true>(lutp, S, r, g, b);
      if (VAR == 6) eval_pair<false, true>(lutp, S, r, g, b);
      if (VAR == 7) eval_scalar<true, false, true>(sm, S, r, g, b);
      if (VAR == 10) eval_cell<true>(lutc, S, r, g, b);
      if (VAR == 11) eval_cell21(lutq, S, r, g, b);
      if (VAR == 8) eval_f4<true>([&](int i) { return sm4[i]; }, S, r, g, b);
      u.e[3 * j] = E<T>::st(r); u.e[3 * j + 1] = E<T>::st(g); u.e[3 * j + 2] = E<T>::st(b);
    }
    uint4* dst = reinterpret_cast<uint4*>(out + grp * PX * 3);
    dst[0] = u.q[0]; dst[1] = u.q[1]; dst[2] = u.q[2];
  }
}

// ---- variant 12/13: one thread per ELEMENT (pixel, channel); channel-planar cell = 3 sectors of 8 corners; the three lanes of a
// pixel read three sectors of the same cell -> one 128-byte line (STRIDE 32, padded) or at most two (STRIDE 24) per pixel ------------
template <typename T, int STRIDE>
__global__ void __launch_bounds__(256) k_lut_elem(const T* __restrict__ in, T* __restrict__ out, int64_t npix, const float* __restrict__ lute, int S) {
  const int64_t nel = npix * 3;
  const float smax = (float)(S - 1);
  for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < nel; e += (int64_t)gridDim.x * 256) {
    const int64_t px = e / 3;
    const int ch = (int)(e - px * 3);
    const T* s = in + px * 3;
    float r = E<T>::ld(__ldg(s)), g = E<T>::ld(__ldg(s + 1)), b = E<T>::ld(__ldg(s + 2));
    Idx q;
    coord<false>(r, smax, S, q.r0, q.r1, q.fr); coord<false>(g, smax, S, q.g0, q.g1, q.fg); coord<false>(b, smax, S, q.b0, q.b1, q.fb);
    const float* p = lute + (size_t)((q.b0 * S + q.g0) * S + q.r0) * STRIDE + ch * 8;
    F8 a = ld256(p);   // c000 c100 c010 c110 c001 c101 c011 c111 of this channel
    float omb = 1.f - q.fb, omg = 1.f - q.fg, omr = 1.f - q.fr;
    float c00 = lerp1<true>(a.a.x, a.b.x, q.fb, omb), c10 = lerp1<true>(a.a.y, a.b.y, q.fb, omb);
    float c01 = lerp1<true>(a.a.z, a.b.z, q.fb, omb), c11 = lerp1<true>(a.a.w, a.b.w, q.fb, omb);
    out[e] = E<T>::st(clamp01(lerp1<true>(lerp1<true>(c00, c01, q.fg, omg), lerp1<true>(c10, c11, q.fg, omg), q.fr, omr)));
  }
}

// ---- variant 14: one lane per PIXEL as in the product, but the gather is cooperative: in round k the three lanes of a group
// all work on the pixel of lane 3g+k (rgb broadcast by 3 shuffles), each loads ONE sector of that pixel's cell and interpolates
// its channel; 3 shuffles hand the results back to the owner.  Same wavefront saving as v13 without a per-element data layout. ----
template <typename T>
__global__ void __launch_bounds__(256) k_lut_coop(const T* __restrict__ in, T* __restrict__ out, int64_t npix, const float* __restrict__ lute, int S) {
  const float smax = (float)(S - 1);
  const int lane = threadIdx.x & 31, grp3 = (lane / 3) * 3, ch = lane - grp3;
  const int64_t nround = (npix + 29) / 30;                      // 30 pixels per warp pass (lanes 30, 31 idle)
  const int64_t warp0 = ((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * 256) >> 5;
  for (int64_t w = warp0; w < nround; w += nwarps) {
    const int64_t px = w * 30 + lane;
    const bool own = lane < 30 && px < npix;
    float r = 0.f, g = 0.f, b = 0.f;
    if (own) { const T* s = in + px * 3; r = E<T>::ld(__ldg(s)); g = E<T>::ld(__ldg(s + 1)); b = E<T>::ld(__ldg(s + 2)); }
    float res[3];
    F8 q[3]; float fr[3], fg[3], fb[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int src = min(grp3 + k, 31);
      const float pr = __shfl_sync(0xffffffffu, r, src), pg = __shfl_sync(0xffffffffu, g, src), pb = __shfl_sync(0xffffffffu, b, src);
      Idx c;
      coord<false>(pr, smax, S, c.r0, c.r1, c.fr); coord<false>(pg, smax, S, c.g0, c.g1, c.fg); coord<false>(pb, smax, S, c.b0, c.b1, c.fb);
      fr[k] = c.fr; fg[k] = c.fg; fb[k] = c.fb;
      q[k] = ld256(lute + (size_t)((c.b0 * S + c.g0) * S + c.r0) * 24 + (ch < 3 ? ch : 0) * 8);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const F8& a = q[k];
      const float omb = 1.f - fb[k], omg = 1.f - fg[k], omr = 1.f - fr[k];
      const float c00 = lerp1<true>(a.a.x, a.b.x, fb[k], omb), c10 = lerp1<true>(a.a.y, a.b.y, fb[k], omb);
      const float c01 = lerp1<true>(a.a.z, a.b.z, fb[k], omb), c11 = lerp1<true>(a.a.w, a.b.w, fb[k], omb);
      res[k] = clamp01(lerp1<true>(lerp1<true>(c00, c01, fg[k], omg), lerp1<true>(c10, c11, fg[k], omg), fr[k], omr));
    }
    // owner lane 3g+k needs channel c of round k from lane 3g+c
    float o[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int src = min(grp3 + c, 31);
      const float v0 = __shfl_sync(0xffffffffu, res[0], src), v1 = __shfl_sync(0xffffffffu, res[1], src), v2 = __shfl_sync(0xffffffffu, res[2], src);
      o[c] = ch == 0 ? v0 : (ch == 1 ? v1 : v2);
    }
    if (own) { T* d = out + px * 3; d[0] = E<T>::st(o[0]); d[1] = E<T>::st(o[1]); d[2] = E<T>::st(o[2]); }
  }
}

template <typename T>
void run_coop(const char* name, const char* tname, const T* in, T* out, int64_t npix, const float* le, int S, int sms, const char* dist, const T* check) {
  auto kern = k_lut_coop<T>;
  cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 0);
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 256, 0));
  int grid = sms * (occ > 0 ? occ : 1) * 4;
  cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  for (int i = 0; i < 2; ++i) kern<<<grid, 256>>>(in, out, npix, le, S);
  CK(cudaDeviceSynchronize());
  float best = 1e9f;
  for (int i = 0; i < 5; ++i) {
    CK(cudaEventRecord(a)); kern<<<grid, 256>>>(in, out, npix, le, S); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
    float ms; CK(cudaEventElapsedTime(&ms, a, b)); best = fminf(best, ms);
  }
  size_t n = 3 << 18;
  std::vector<T> h1(n), h2(n);
  CK(cudaMemcpy(h1.data(), out, n * sizeof(T), cudaMemcpyDeviceToHost)); CK(cudaMemcpy(h2.data(), check, n * sizeof(T), cudaMemcpyDeviceToHost));
  double md = 0; for (size_t i = 0; i < n; ++i) md = fmax(md, fabs((double)(float)h1[i] - (double)(float)h2[i]));
  double gpx = npix / (best * 1e-3) / 1e9;
  printf("{\"variant\": \"%s\", \"dtype\": \"%s\", \"dist\": \"%s\", \"S\": %d, \"ms\": %.4f, \"Gpx/s\": %.1f, \"GB/s\": %.0f, \"occ\": %d, \"maxdiff_vs_v1\": %.3g}\n",
         name, tname, dist, S, best, gpx, gpx * 6 * sizeof(T), occ, md);
  fflush(stdout);
}

template <typename T, int STRIDE>
void run_elem(const char* name, const char* tname, const T* in, T* out, int64_t npix, const float* le, int S, int sms, const char* dist, const T* check) {
  auto kern = k_lut_elem<T, STRIDE>;
  cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 0);
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 256, 0));
  int grid = sms * (occ > 0 ? occ : 1) * 4;
  cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  for (int i = 0; i < 2; ++i) kern<<<grid, 256>>>(in, out, npix, le, S);
  CK(cudaDeviceSynchronize());
  float best = 1e9f;
  for (int i = 0; i < 5; ++i) {
    CK(cudaEventRecord(a)); kern<<<grid, 256>>>(in, out, npix, le, S); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
    float ms; CK(cudaEventElapsedTime(&ms, a, b)); best = fminf(best, ms);
  }
  size_t n = 3 << 18;
  std::vector<T> h1(n), h2(n);
  CK(cudaMemcpy(h1.data(), out, n * sizeof(T), cudaMemcpyDeviceToHost)); CK(cudaMemcpy(h2.data(), check, n * sizeof(T), cudaMemcpyDeviceToHost));
  double md = 0; for (size_t i = 0; i < n; ++i) md = fmax(md, fabs((double)(float)h1[i] - (double)(float)h2[i]));
  double gpx = npix / (best * 1e-3) / 1e9;
  printf("{\"variant\": \"%s\", \"dtype\": \"%s\", \"dist\": \"%s\", \"S\": %d, \"ms\": %.4f, \"Gpx/s\": %.1f, \"GB/s\": %.0f, \"occ\": %d, \"maxdiff_vs_v1\": %.3g}\n",
         name, tname, dist, S, best, gpx, gpx * 6 * sizeof(T), occ, md);
  fflush(stdout);
}

template <typename T> __global__ void k_fill(T* p, int64_t npix, int W, int H, int mode, uint32_t seed) {
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < npix; i += (int64_t)gridDim.x * 256) {
    int x = (int)(i % W), y = (int)((i / W) % H);
    uint32_t h = (uint32_t)i * 2654435761u + seed; h ^= h >> 15; h *= 2246822519u; h ^= h >> 13; h *= 3266489917u; h ^= h >> 16;
    float n0 = (h & 0xffff) / 65536.f, n1 = (h >> 16) / 65536.f, n2 = ((h * 747796405u) >> 16) / 65536.f;
    float r, g, b;
    if (mode == 0) { r = n0; g = n1; b = n2; }
    else {
      r = 0.5f + 0.25f * __sinf(x * 0.011f + 0.3f) + 0.2f * __sinf(y * 0.013f) + 0.02f * (n0 - 0.5f);
      g = 0.5f + 0.25f * __sinf(x * 0.007f + 1.3f) + 0.2f * __sinf(y * 0.017f + 0.5f) + 0.02f * (n1 - 0.5f);
      b = 0.45f + 0.25f * __sinf(x * 0.005f + 2.1f) + 0.2f * __sinf(y * 0.009f + 1.5f) + 0.02f * (n2 - 0.5f);
    }
    if (mode == 2) {   // natural + film-grain-like Gaussian noise (sigma 0.08 / 0.04 / 0.12): what the LUT sees after FastFilmGrain
      float u1 = (n0 * 65535.f + 1.f) / 65537.f, rr = sqrtf(-2.f * __logf(u1));
      float u2 = (n2 * 65535.f + 1.f) / 65537.f, r2 = sqrtf(-2.f * __logf(u2));
      r += 0.08f * rr * __cosf(6.2831853f * n1); g += 0.04f * rr * __sinf(6.2831853f * n1); b += 0.12f * r2 * __cosf(6.2831853f * n0);
    }
    p[i * 3] = E<T>::st(clamp01(r)); p[i * 3 + 1] = E<T>::st(clamp01(g)); p[i * 3 + 2] = E<T>::st(clamp01(b));
  }
}

template <typename T, int VAR>
void run(const char* name, const char* tname, const T* in, T* out, int64_t npix, const float* l3, const float4* l4, const float* lp, int S,
         size_t smem, int sms, const char* dist, const T* check, const float* lc = nullptr, const float* lq = nullptr) {
  auto kern = k_lut<T, VAR>;
  if (smem > 48 * 1024) CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  if (smem == 0) cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 0);
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 256, smem));
  int grid = sms * (occ > 0 ? occ : 1) * (smem ? 1 : 4);
  cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  for (int i = 0; i < 2; ++i) kern<<<grid, 256, smem>>>(in, out, npix, l3, l4, lp, S, lc, lq);
  CK(cudaDeviceSynchronize());
  float best = 1e9f;
  for (int i = 0; i < 5; ++i) {
    CK(cudaEventRecord(a)); kern<<<grid, 256, smem>>>(in, out, npix, l3, l4, lp, S, lc, lq); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
    float ms; CK(cudaEventElapsedTime(&ms, a, b)); best = fminf(best, ms);
  }
  // max diff vs the reference variant's output (first 1M elements)
  double md = -1;
  if (check) {
    size_t n = 3 << 18;
    std::vector<T> h1(n), h2(n);
    CK(cudaMemcpy(h1.data(), out, n * sizeof(T), cudaMemcpyDeviceToHost)); CK(cudaMemcpy(h2.data(), check, n * sizeof(T), cudaMemcpyDeviceToHost));
    md = 0; for (size_t i = 0; i < n; ++i) md = fmax(md, fabs((double)(float)h1[i] - (double)(float)h2[i]));
  }
  double gpx = npix / (best * 1e-3) / 1e9;
  printf("{\"variant\": \"%s\", \"dtype\": \"%s\", \"dist\": \"%s\", \"S\": %d, \"ms\": %.4f, \"Gpx/s\": %.1f, \"GB/s\": %.0f, \"occ\": %d, \"maxdiff_vs_v1\": %.3g}\n",
         name, tname, dist, S, best, gpx, gpx * 6 * sizeof(T), occ, md);
  fflush(stdout);
}

template <typename T> void suite(const char* tname, int sms) {
  const int W = 3840, H = 2160, B = (sizeof(T) == 4) ? 4 : 8;
  const int64_t npix = (int64_t)B * W * H;
  T *in, *out, *ref;
  CK(cudaMalloc(&in, npix * 3 * sizeof(T))); CK(cudaMalloc(&out, npix * 3 * sizeof(T))); CK(cudaMalloc(&ref, npix * 3 * sizeof(T)));
  for (int S : {33, 17}) {
    size_t n = (size_t)S * S * S;
    std::vector<float> h3(n * 3), hp(n * 8, 0.f); std::vector<float4> h4(n);
    for (int b = 0; b < S; ++b) for (int g = 0; g < S; ++g) for (int r = 0; r < S; ++r) {
      size_t i = ((size_t)b * S + g) * S + r;
      float fr = r / (float)(S - 1), fg = g / (float)(S - 1), fb = b / (float)(S - 1);
      float y = 0.2126f * fr + 0.7152f * fg + 0.0722f * fb;
      float v[3] = {0.06f + 0.9f * (y + 0.72f * (fr - y)) * 1.03f, 0.05f + 0.9f * (y + 0.72f * (fg - y)), 0.07f + 0.85f * (y + 0.72f * (fb - y))};
      for (int c = 0; c < 3; ++c) { v[c] = roundf(fminf(fmaxf(v[c], 0.f), 1.f) * 1e6f) / 1e6f; h3[i * 3 + c] = v[c]; }
      h4[i] = make_float4(v[0], v[1], v[2], 0.f);
    }
    for (int b = 0; b < S; ++b) for (int g = 0; g < S; ++g) for (int r = 0; r < S; ++r) {
      size_t i = ((size_t)b * S + g) * S + r, i1 = ((size_t)b * S + g) * S + (r + 1 < S ? r + 1 : S - 1);
      for (int c = 0; c < 3; ++c) { hp[i * 8 + c] = h3[i * 3 + c]; hp[i * 8 + 4 + c] = h3[i1 * 3 + c]; }
    }
    std::vector<float> hc(n * 24, 0.f);
    for (int b = 0; b < S; ++b) for (int g = 0; g < S; ++g) for (int r = 0; r < S; ++r) {
      size_t i = ((size_t)b * S + g) * S + r;
      int b1 = b + 1 < S ? b + 1 : S - 1, g1 = g + 1 < S ? g + 1 : S - 1, r1 = r + 1 < S ? r + 1 : S - 1;
      int cb[8] = {b, b, b, b, b1, b1, b1, b1}, cg[8] = {g, g, g1, g1, g, g, g1, g1}, cr[8] = {r, r1, r, r1, r, r1, r, r1};
      for (int k = 0; k < 8; ++k) for (int c = 0; c < 3; ++c) hc[i * 24 + k * 3 + c] = h3[(((size_t)cb[k] * S + cg[k]) * S + cr[k]) * 3 + c];
    }
    std::vector<uint32_t> hq(n * 16, 0u);
    for (size_t i = 0; i < n; ++i) for (int k = 0; k < 8; ++k) {
      uint32_t q[3];
      for (int c = 0; c < 3; ++c) q[c] = (uint32_t)llround((double)hc[i * 24 + k * 3 + c] * 2097151.0);   // unorm21 (scale 2^21-1 ~ 2^21)
      hq[i * 16 + 2 * k] = q[0] | (q[1] << 21);
      hq[i * 16 + 2 * k + 1] = (q[1] >> 11) | (q[2] << 10);
    }
    std::vector<float> he32(n * 32, 0.f), he24(n * 24, 0.f);
    for (size_t i = 0; i < n; ++i) for (int k = 0; k < 8; ++k) for (int c = 0; c < 3; ++c) {
      he32[i * 32 + c * 8 + k] = hc[i * 24 + k * 3 + c];
      he24[i * 24 + c * 8 + k] = hc[i * 24 + k * 3 + c];
    }
    float *le32, *le24;
    CK(cudaMalloc(&le32, n * 128)); CK(cudaMemcpy(le32, he32.data(), n * 128, cudaMemcpyHostToDevice));
    CK(cudaMalloc(&le24, n * 96)); CK(cudaMemcpy(le24, he24.data(), n * 96, cudaMemcpyHostToDevice));
    float* lq; CK(cudaMalloc(&lq, n * 64)); CK(cudaMemcpy(lq, hq.data(), n * 64, cudaMemcpyHostToDevice));
    float *l3, *lp, *lc; float4* l4;
    CK(cudaMalloc(&l3, n * 12)); CK(cudaMalloc(&l4, n * 16)); CK(cudaMalloc(&lp, n * 32)); CK(cudaMalloc(&lc, n * 96));
    CK(cudaMemcpy(lc, hc.data(), n * 96, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(l3, h3.data(), n * 12, cudaMemcpyHostToDevice)); CK(cudaMemcpy(l4, h4.data(), n * 16, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(lp, hp.data(), n * 32, cudaMemcpyHostToDevice));
    for (int mode = 2; mode >= 0; --mode) {
      const char* dist = mode == 2 ? "natural+grain" : (mode ? "natural" : "white");
      k_fill<T><<<sms * 8, 256>>>(in, npix, W, H, mode, 12345u);
      CK(cudaDeviceSynchronize());
      if (S == 33 && mode == 1) run<T, 9>("io_only", tname, in, out, npix, l3, l4, lp, S, 0, sms, dist, nullptr);
      run<T, 1>("v1_scalar_exact", tname, in, ref, npix, l3, l4, lp, S, 0, sms, dist, nullptr);
      run<T, 0>("v0_scalar_exact_div", tname, in, out, npix, l3, l4, lp, S, 0, sms, dist, ref);
      run<T, 2>("v2_f4_exact", tname, in, out, npix, l3, l4, lp, S, 0, sms, dist, ref);
      run<T, 3>("v3_f4_fast", tname, in, out, npix, l3, l4, lp, S, 0, sms, dist, ref);
      run<T, 4>("v4_pair_2x128_exact", tname, in, out, npix, l3, l4, lp, S, 0, sms, dist, ref);
      run<T, 5>("v5_pair_256_exact", tname, in, out, npix, l3, l4, lp, S, 0, sms, dist, ref);
      run<T, 6>("v6_pair_256_fast", tname, in, out, npix, l3, l4, lp, S, 0, sms, dist, ref);
      run<T, 10>("v10_cell_3x256_exact", tname, in, out, npix, l3, l4, lp, S, 0, sms, dist, ref, lc);
      run<T, 11>("v11_cell_u21_2x256", tname, in, out, npix, l3, l4, lp, S, 0, sms, dist, ref, lc, lq);
      run_elem<T, 32>("v12_elem_planar_pad128", tname, in, out, npix, le32, S, sms, dist, ref);
      run_elem<T, 24>("v13_elem_planar_96", tname, in, out, npix, le24, S, sms, dist, ref);
      run_coop<T>("v14_pixel_owner_3lane_coop", tname, in, out, npix, le24, S, sms, dist, ref);
      if (n * 12 <= 200 * 1024) run<T, 7>("v7_smem_scalar_exact", tname, in, out, npix, l3, l4, lp, S, n * 12, sms, dist, ref);
      if (n * 16 <= 200 * 1024) run<T, 8>("v8_smem_f4_exact", tname, in, out, npix, l3, l4, lp, S, n * 16, sms, dist, ref);
    }
    cudaFree(l3); cudaFree(l4); cudaFree(lp); cudaFree(lc); cudaFree(lq); cudaFree(le32); cudaFree(le24);
  }
  cudaFree(in); cudaFree(out); cudaFree(ref);
}

int main() {
  int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  suite<float>("f32", sms);
  suite<__half>("f16", sms);
  return 0;
}

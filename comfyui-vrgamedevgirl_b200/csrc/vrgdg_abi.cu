// vrgdg_abi.cu — extern "C" boundary of libvrgdg_b200.so (declared in include/vrgdg_b200.h).
// Validates arguments, builds TMA tensor maps, dispatches on dtype, never throws.
#include "../../include/vrgdg_b200.h"
#include "vrgdg_kernels.cuh"
#include <cmath>
#include "vrgdg_adjust.cuh"
#include "vrgdg_resize.cuh"
#include "vrgdg_lanczos.cuh"
#include "vrgdg_temporal.cuh"
#include "vrgdg_histmatch.cuh"
#include <atomic>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace vrgdg {
static std::atomic<int64_t> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
}  // namespace vrgdg

using namespace vrgdg;

namespace {

thread_local char t_err[512] = "";
thread_local const char* t_tile_path = "none";

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_err, sizeof(t_err), fmt, ap);
  va_end(ap);
  return code;
}
int fail_cuda(cudaError_t e, const char* where) {
  return fail(VRGDG_E_CUDA, "%s: %s (%s)", where, cudaGetErrorName(e), cudaGetErrorString(e));
}

size_t elem_size(int dtype) { return dtype == VRGDG_F32 ? 4 : (dtype == VRGDG_U8BGR ? 1 : 2); }
bool dtype_ok(int dtype) { return dtype == VRGDG_F32 || dtype == VRGDG_F16 || dtype == VRGDG_BF16 || dtype == VRGDG_U8BGR; }

int get_ctx(void* stream, LaunchCtx& ctx) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return fail_cuda(e, "cudaGetDevice");
  static thread_local int cached_dev = -1, cached_sms = 0, cached_major = 0, cached_minor = 0;
  if (cached_dev != dev) {
    int sms = 0, major = 0, minor = 0;
    if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return fail_cuda(e, "cudaDeviceGetAttribute");
    if ((e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev)) != cudaSuccess) return fail_cuda(e, "cudaDeviceGetAttribute");
    if ((e = cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev)) != cudaSuccess) return fail_cuda(e, "cudaDeviceGetAttribute");
    cached_dev = dev; cached_sms = sms; cached_major = major; cached_minor = minor;
  }
  if (cached_major != 9 || cached_minor != 0)   // sm_90a code runs on compute capability 9.0 only
    return fail(VRGDG_E_UNSUPPORTED, "libvrgdg_b200 holds sm_90a code only; device %d has compute capability %d.%d", dev, cached_major,
                cached_minor);
  ctx.stream = reinterpret_cast<cudaStream_t>(stream);
  ctx.sms = cached_sms;
  return VRGDG_OK;
}

int check_frames(const void* in, const void* out, int B, int H, int W, int dtype, const char* who) {
  if (!dtype_ok(dtype)) return fail(VRGDG_E_INVALID, "%s: unknown dtype %d", who, dtype);
  if (B < 0 || H < 0 || W < 0) return fail(VRGDG_E_INVALID, "%s: negative shape [%d,%d,%d]", who, B, H, W);
  if ((int64_t)H * W >= (int64_t)1 << 31) return fail(VRGDG_E_UNSUPPORTED, "%s: frame of %d x %d pixels exceeds 2^31", who, H, W);
  if ((int64_t)B * H * W == 0) return VRGDG_OK;
  if (!in || !out) return fail(VRGDG_E_INVALID, "%s: null frame pointer", who);
  size_t es = elem_size(dtype);
  if ((reinterpret_cast<uintptr_t>(in) % es) || (reinterpret_cast<uintptr_t>(out) % es))
    return fail(VRGDG_E_ALIGN, "%s: frame pointer not aligned to its element size", who);
  return VRGDG_OK;
}

#define DISPATCH_DTYPE(dtype, CALL)                                        \
  ((dtype) == VRGDG_F32 ? CALL(float) : ((dtype) == VRGDG_F16 ? CALL(__half) : ((dtype) == VRGDG_BF16 ? CALL(__nv_bfloat16) : CALL(uint8_t))))

// ---- TMA tensor map over frames [B][H][RW] ---------------------------------------------------------
typedef CUresult (*encode_fn_t)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

encode_fn_t get_encode() {
  static encode_fn_t fn = []() -> encode_fn_t {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) != cudaSuccess ||
        qr != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<encode_fn_t>(p);
  }();
  return fn;
}

// returns true when a map was built (TMA path usable)
bool build_tmap(CUtensorMap* map, const void* in, int B, int H, int RW, int dtype, int box_x, int box_y) {
  const size_t es = elem_size(dtype);
  if (getenv("VRGDG_NO_TMA")) return false;
  if ((reinterpret_cast<uintptr_t>(in) & 15u) || ((size_t)RW * es) % 16 != 0) return false;
  if (RW < box_x || H < box_y) return false;      // tiny frames take the generic loader
  encode_fn_t enc = get_encode();
  if (!enc) return false;
  CUtensorMapDataType dt = dtype == VRGDG_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                         : dtype == VRGDG_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                         : dtype == VRGDG_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8;
  cuuint64_t dims[3] = {(cuuint64_t)RW, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[2] = {(cuuint64_t)RW * es, (cuuint64_t)RW * es * (cuuint64_t)H};
  cuuint32_t box[3] = {(cuuint32_t)box_x, (cuuint32_t)box_y, 1u};
  cuuint32_t estr[3] = {1u, 1u, 1u};
  CUresult r = enc(map, dt, 3, const_cast<void*>(in), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

size_t lut_cells_floats(int S) { return (size_t)S * S * S * LUT_CELL_FLOATS; }
// packed table = corner cells (96 B per node) followed by the polynomial cells of the fast chains (96 B per node, vrgdg_math.cuh)

void fill_lut(LutParams& L, const float* lut, int S, const float* dmin, const float* dspan, float blend, float omb) {
  L.lut = lut; L.S = S; L.smax = (float)(S - 1);
  L.lutp = lut + lut_cells_floats(S);
  for (int i = 0; i < 3; ++i) { L.dmin[i] = dmin[i]; L.dspan[i] = dspan[i]; }
  L.blend = blend; L.one_minus_blend = omb;
  L.unit_domain = (dmin[0] == 0.f && dmin[1] == 0.f && dmin[2] == 0.f && dspan[0] == 1.f && dspan[1] == 1.f && dspan[2] == 1.f) ? 1 : 0;
}

void zero_point(PointParams& P, int B, int H, int W) {
  memset(&P, 0, sizeof(P));
  P.B = B; P.H = H; P.W = W; P.hw = (int64_t)H * W;
}

int run_tile(const void* in, void* out, int B, int H, int W, int dtype, TileParams& Q, int mask, bool exact, const LaunchCtx& ctx) {
  if (in == out) return fail(VRGDG_E_INVALID, "tile kernels cannot run in place (in == out)");
  Q.B = B; Q.H = H; Q.W = W; Q.RW = 3 * W;
  int bx = 0, by = 0;
#define GEO(T) (tile_geometry<T>(H, Q.RW, Q.tiles_x, Q.tiles_y, bx, by), 0)
  (void)DISPATCH_DTYPE(dtype, GEO);
#undef GEO
  Q.total_tiles = (int64_t)B * Q.tiles_x * Q.tiles_y;
  if (Q.total_tiles >= ((int64_t)1 << 31)) return fail(VRGDG_E_UNSUPPORTED, "batch of %d frames has too many tiles for one launch; split it", B);
  CUtensorMap map;
  bool tma = build_tmap(&map, in, B, H, Q.RW, dtype, bx, by);
  Q.use_tma = tma ? 1 : 0;
  const size_t es = elem_size(dtype);
  Q.vec_store = (((size_t)Q.RW * es) % 16 == 0 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0) ? 1 : 0;
  t_tile_path = tma ? "tma" : "generic";
#define TL(T) launch_tile<T>(tma ? &map : nullptr, in, out, Q, mask, exact, ctx)
  cudaError_t e = DISPATCH_DTYPE(dtype, TL);
#undef TL
  if (e != cudaSuccess) return fail_cuda(e, "k_tile launch");
  return VRGDG_OK;
}

int check_lut(const float* lut, int S, const float* dmin, const float* dspan, const char* who) {
  if (!lut || !dmin || !dspan) return fail(VRGDG_E_INVALID, "%s: null LUT / domain pointer", who);
  if (S < 2 || S > 256) return fail(VRGDG_E_INVALID, "%s: LUT size %d outside [2,256]", who, S);
  if (reinterpret_cast<uintptr_t>(lut) & 31u) return fail(VRGDG_E_ALIGN, "%s: packed LUT must be 32-byte aligned", who);
  return VRGDG_OK;
}

}  // namespace

extern "C" {

int vrgdg_version(void) { return VRGDG_ABI_VERSION; }
const char* vrgdg_last_error(void) { return t_err; }
int64_t vrgdg_launch_count(void) { return g_launches.load(); }
const char* vrgdg_last_tile_path(void) { return t_tile_path; }

int vrgdg_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return fail_cuda(e, "cudaGetDevice");
  int v = 0;
  if (sm_count) { if ((e = cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return fail_cuda(e, "attr"); *sm_count = v; }
  if (cc_major) { if ((e = cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, dev)) != cudaSuccess) return fail_cuda(e, "attr"); *cc_major = v; }
  if (cc_minor) { if ((e = cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, dev)) != cudaSuccess) return fail_cuda(e, "attr"); *cc_minor = v; }
  return VRGDG_OK;
}

int64_t vrgdg_lut3d_packed_bytes(int lut_size) {
  if (lut_size < 2 || lut_size > 256) return 0;
  return (int64_t)lut_cells_floats(lut_size) * 2 * 4;
}

int vrgdg_lut3d_pack(const float* lut, float* packed, int lut_size, void* stream) {
  if (!lut || !packed) return fail(VRGDG_E_INVALID, "vrgdg_lut3d_pack: null pointer");
  if (lut_size < 2 || lut_size > 256) return fail(VRGDG_E_INVALID, "vrgdg_lut3d_pack: LUT size %d outside [2,256]", lut_size);
  if (reinterpret_cast<uintptr_t>(packed) & 31u) return fail(VRGDG_E_ALIGN, "vrgdg_lut3d_pack: packed buffer must be 32-byte aligned");
  LaunchCtx ctx;
  int rc = get_ctx(stream, ctx);
  if (rc) return rc;
  const int n = lut_size * lut_size * lut_size;
  k_lut_pack<<<(n + 255) / 256, 256, 0, ctx.stream>>>(lut, packed, lut_size);
  count_launch();
  k_lutp_pack<<<(n + 255) / 256, 256, 0, ctx.stream>>>(lut, packed + lut_cells_floats(lut_size), lut_size);
  count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_lut3d_pack");
  return VRGDG_OK;
}

int vrgdg_lut3d_apply(const void* in, void* out, int64_t npix, int channels, int dtype, const float* lut, int lut_size,
                      const float* dmin_host, const float* dspan_host, float blend, float one_minus_blend, void* stream) {
  if (!dtype_ok(dtype)) return fail(VRGDG_E_INVALID, "vrgdg_lut3d_apply: unknown dtype %d", dtype);
  if (channels != 3 && channels != 4) return fail(VRGDG_E_INVALID, "vrgdg_lut3d_apply: channels must be 3 or 4, got %d", channels);
  if (npix < 0) return fail(VRGDG_E_INVALID, "vrgdg_lut3d_apply: negative pixel count");
  if (!(blend > 0.0f) || blend > 1.0f) return fail(VRGDG_E_INVALID, "vrgdg_lut3d_apply: blend %g outside (0,1]", blend);
  int rc = check_lut(lut, lut_size, dmin_host, dspan_host, "vrgdg_lut3d_apply");
  if (rc) return rc;
  if (npix == 0) return VRGDG_OK;
  if (!in || !out) return fail(VRGDG_E_INVALID, "vrgdg_lut3d_apply: null frame pointer");
  LaunchCtx ctx;
  if ((rc = get_ctx(stream, ctx))) return rc;
  LutParams L;
  fill_lut(L, lut, lut_size, dmin_host, dspan_host, blend, one_minus_blend);
  cudaError_t e;
  if (channels == 4 && dtype == VRGDG_U8BGR) return fail(VRGDG_E_UNSUPPORTED, "vrgdg_lut3d_apply: 4-channel uint8 frames are not supported");
  if (channels == 4) {
#define LR(T) launch_lut_rgba<T>(in, out, npix, L, ctx)
    e = DISPATCH_DTYPE(dtype, LR);
#undef LR
  } else {
    // frames are independent of shape here: treat the pixel stream as frames of <= 2^30 pixels
    // (chunk divisible by 8 keeps the vector path for every chunk but the last)
    const int64_t chunk = (int64_t)1 << 30;
    e = cudaSuccess;
    for (int64_t p0 = 0; p0 < npix && e == cudaSuccess; p0 += chunk) {
      int64_t n = npix - p0 < chunk ? npix - p0 : chunk;
      PointParams P;
      zero_point(P, 1, 1, (int)n);
      P.lut = L;
      const char* ip = reinterpret_cast<const char*>(in) + p0 * 3 * elem_size(dtype);
      char* op = reinterpret_cast<char*>(out) + p0 * 3 * elem_size(dtype);
#define PT(T) launch_point<T>(ip, op, P, ST_LUT, true, ctx)
      e = DISPATCH_DTYPE(dtype, PT);
#undef PT
    }
  }
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_lut3d_apply");
  return VRGDG_OK;
}

int vrgdg_grain(const void* in, void* out, int B, int H, int W, int dtype, float intensity, float sat, float one_minus_sat,
                uint64_t seed, int64_t frame0, int seed_mode, const void* ext_noise, void* stream) {
  int rc = check_frames(in, out, B, H, W, dtype, "vrgdg_grain");
  if (rc) return rc;
  if (seed_mode != VRGDG_SEED_PER_CLIP && seed_mode != VRGDG_SEED_PER_FRAME) return fail(VRGDG_E_INVALID, "vrgdg_grain: bad seed_mode %d", seed_mode);
  if ((int64_t)B * H * W == 0) return VRGDG_OK;
  LaunchCtx ctx;
  if ((rc = get_ctx(stream, ctx))) return rc;
  PointParams P;
  zero_point(P, B, H, W);
  P.gI = intensity; P.gs = sat; P.goms = one_minus_sat;
  P.seed = seed; P.frame0 = frame0; P.seed_mode = seed_mode; P.ext_noise = ext_noise;
  grain_make_key(seed, seed_mode, P.gkey);
  const bool exact = ext_noise != nullptr;
#define PT(T) launch_point<T>(in, out, P, ST_GRAIN, exact, ctx)
  cudaError_t e = DISPATCH_DTYPE(dtype, PT);
#undef PT
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_grain");
  return VRGDG_OK;
}

int vrgdg_grain_noise(float* out, int B, int H, int W, uint64_t seed, int64_t frame0, int seed_mode, void* stream) {
  if (B < 0 || H < 0 || W < 0) return fail(VRGDG_E_INVALID, "vrgdg_grain_noise: negative shape");
  if ((int64_t)B * H * W == 0) return VRGDG_OK;
  if (!out) return fail(VRGDG_E_INVALID, "vrgdg_grain_noise: null output");
  LaunchCtx ctx;
  int rc = get_ctx(stream, ctx);
  if (rc) return rc;
  int64_t total = (int64_t)B * H * W;
  int grid = (int)(((total + 255) / 256) < (int64_t)ctx.sms * 16 ? ((total + 255) / 256) : (int64_t)ctx.sms * 16);
  if (seed_mode != VRGDG_SEED_PER_CLIP && seed_mode != VRGDG_SEED_PER_FRAME) return fail(VRGDG_E_INVALID, "vrgdg_grain_noise: bad seed_mode %d", seed_mode);
  GrainKey K;
  grain_make_key(seed, seed_mode, K);
  k_grain_noise<<<grid, 256, 0, ctx.stream>>>(out, B, W, (int64_t)H * W, seed, frame0, seed_mode, K);
  count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_grain_noise");
  return VRGDG_OK;
}

int vrgdg_stencil3x3(const void* in, void* out, int B, int H, int W, int dtype, int op, float strength, int border, void* stream) {
  int rc = check_frames(in, out, B, H, W, dtype, "vrgdg_stencil3x3");
  if (rc) return rc;
  if (op < VRGDG_STENCIL_BOX_UNSHARP || op > VRGDG_STENCIL_SOBEL_GPU) return fail(VRGDG_E_INVALID, "vrgdg_stencil3x3: bad op %d", op);
  if (border != VRGDG_BORDER_REPLICATE && border != VRGDG_BORDER_ZERO) return fail(VRGDG_E_INVALID, "vrgdg_stencil3x3: bad border %d", border);
  if ((int64_t)B * H * W == 0) return VRGDG_OK;
  LaunchCtx ctx;
  if ((rc = get_ctx(stream, ctx))) return rc;
  TileParams Q;
  memset(&Q, 0, sizeof(Q));
  zero_point(Q.P, B, H, W);
  Q.op = op; Q.strength = strength; Q.border = border;
  Q.exact_stencil = (dtype == VRGDG_F32 || dtype == VRGDG_U8BGR) ? 1 : 0;   // fp32 / byte frames: bit-identical to the NumPy nodes; 16-bit frames round once anyway
  return run_tile(in, out, B, H, W, dtype, Q, 0, true, ctx);
}

int64_t vrgdg_lab_moments_scratch_bytes(int B) {
  if (B < 0) return 0;
  return (int64_t)B * MOMENT_BLOCKS * 6 * (int64_t)sizeof(double);
}

static int moments_common(const void* in, int B, int H, int W, int dtype, int row0, int rows, const PointParams* grainP,
                          double* sums, void* scratch, int64_t scratch_bytes, void* stream, const char* who) {
  if (!dtype_ok(dtype)) return fail(VRGDG_E_INVALID, "%s: unknown dtype %d", who, dtype);
  if (B < 0 || H <= 0 || W <= 0) return fail(VRGDG_E_INVALID, "%s: bad shape [%d,%d,%d]", who, B, H, W);
  if (row0 < 0 || rows <= 0 || row0 + rows > H) return fail(VRGDG_E_INVALID, "%s: row range [%d,%d) outside [0,%d)", who, row0, row0 + rows, H);
  if (B == 0) return VRGDG_OK;
  if (!in || !sums || !scratch) return fail(VRGDG_E_INVALID, "%s: null pointer", who);
  if (scratch_bytes < vrgdg_lab_moments_scratch_bytes(B)) return fail(VRGDG_E_INVALID, "%s: scratch too small (%lld < %lld)", who, (long long)scratch_bytes, (long long)vrgdg_lab_moments_scratch_bytes(B));
  if (reinterpret_cast<uintptr_t>(sums) % 8 || reinterpret_cast<uintptr_t>(scratch) % 8) return fail(VRGDG_E_ALIGN, "%s: sums/scratch must be 8-byte aligned", who);
  LaunchCtx ctx;
  int rc = get_ctx(stream, ctx);
  if (rc) return rc;
  PointParams P;
  if (grainP) P = *grainP; else zero_point(P, B, H, W);
#define MO(T) launch_moments<T>(in, P, grainP != nullptr, row0, rows, sums, reinterpret_cast<double*>(scratch), ctx)
  cudaError_t e = DISPATCH_DTYPE(dtype, MO);
#undef MO
  if (e != cudaSuccess) return fail_cuda(e, who);
  return VRGDG_OK;
}

int vrgdg_lab_moments(const void* in, int B, int H, int W, int dtype, int row0, int rows, double* sums, void* scratch,
                      int64_t scratch_bytes, void* stream) {
  return moments_common(in, B, H, W, dtype, row0, rows, nullptr, sums, scratch, scratch_bytes, stream, "vrgdg_lab_moments");
}

int vrgdg_colormatch_params(const double* frame_sums, int B, const double* ref_sums, int n_ref, float* params, void* stream) {
  if (B < 0) return fail(VRGDG_E_INVALID, "vrgdg_colormatch_params: negative B");
  if (B == 0) return VRGDG_OK;
  if (!frame_sums || !ref_sums || !params) return fail(VRGDG_E_INVALID, "vrgdg_colormatch_params: null pointer");
  if (n_ref != 1 && n_ref != B) return fail(VRGDG_E_INVALID, "vrgdg_colormatch_params: reference batch %d is neither 1 nor %d", n_ref, B);
  LaunchCtx ctx;
  int rc = get_ctx(stream, ctx);
  if (rc) return rc;
  k_colormatch_params<<<(B + 127) / 128, 128, 0, ctx.stream>>>(frame_sums, B, ref_sums, n_ref, params);
  count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_colormatch_params");
  return VRGDG_OK;
}

int vrgdg_colormatch_apply(const void* in, void* out, int B, int H, int W, int dtype, const float* params, float t,
                           float one_minus_t, void* stream) {
  int rc = check_frames(in, out, B, H, W, dtype, "vrgdg_colormatch_apply");
  if (rc) return rc;
  if ((int64_t)B * H * W == 0) return VRGDG_OK;
  if (!params) return fail(VRGDG_E_INVALID, "vrgdg_colormatch_apply: null params");
  LaunchCtx ctx;
  if ((rc = get_ctx(stream, ctx))) return rc;
  PointParams P;
  zero_point(P, B, H, W);
  P.cm_params = params; P.cm_t = t; P.cm_omt = one_minus_t;
#define PT(T) launch_point<T>(in, out, P, ST_CM, true, ctx)
  cudaError_t e = DISPATCH_DTYPE(dtype, PT);
#undef PT
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_colormatch_apply");
  return VRGDG_OK;
}

static int chain_point_params(const vrgdg_chain_desc* d, int B, int H, int W, PointParams& P, int& mask, bool& exact, const void* ext_noise, bool fast) {
  zero_point(P, B, H, W);
  mask = 0;
  if (d->grain_enabled) {
    if (d->grain_seed_mode != VRGDG_SEED_PER_CLIP && d->grain_seed_mode != VRGDG_SEED_PER_FRAME) return fail(VRGDG_E_INVALID, "chain: bad grain seed_mode %d", d->grain_seed_mode);
    mask |= ST_GRAIN;
    P.gI = d->grain_intensity; P.gs = d->grain_sat; P.goms = d->grain_one_minus_sat;
    P.seed = d->grain_seed; P.frame0 = d->grain_frame0; P.seed_mode = d->grain_seed_mode;
    grain_make_key(P.seed, P.seed_mode, P.gkey);
    P.ext_noise = ext_noise;
  }
  if (d->colormatch_enabled) {
    if (!d->cm_params) return fail(VRGDG_E_INVALID, "chain: colour match enabled without params");
    mask |= ST_CM;
    P.cm_params = d->cm_params; P.cm_t = d->cm_t; P.cm_omt = d->cm_one_minus_t;
  }
  if (d->lut_enabled) {
    int rc = check_lut(d->lut, d->lut_size, d->lut_dmin, d->lut_dspan, "chain");
    if (rc) return rc;
    if (!(d->lut_blend > 0.0f) || d->lut_blend > 1.0f) return fail(VRGDG_E_INVALID, "chain: LUT blend %g outside (0,1]", d->lut_blend);
    mask |= ST_LUT;
    fill_lut(P.lut, d->lut, d->lut_size, d->lut_dmin, d->lut_dspan, d->lut_blend, d->lut_one_minus_blend);
  }
  // exact arithmetic unless the chain draws its own noise (then only the noise-free stages stay exact in k_point<.., true>)
  exact = !(d->grain_enabled && (ext_noise == nullptr || fast));
  return VRGDG_OK;
}

/* Core of the chain entry points.  from_f: `in` holds the (fx, fy, fz) planes the moments pass stored (fp32, same layout as the
 * frames) and the grain + forward-Lab half of the colour match has already happened: stages become ST_CMF [| ST_LUT].
 * cm_params (when non-null) replaces desc->cm_params; frame_offset is added to both grain frame indices (group scheduling). */
static int chain_apply_core(const void* in, void* out, int B, int H, int W, int dtype, const vrgdg_chain_desc* d,
                            const void* ext_noise, bool fast, void* stream, const float* cm_params, bool from_f, int64_t frame_offset,
                            int grid_limit = 0) {
  if (!d) return fail(VRGDG_E_INVALID, "vrgdg_chain_apply: null descriptor");
  int rc = check_frames(in, out, B, H, W, dtype, "vrgdg_chain_apply");
  if (rc) return rc;
  if (d->stencil_op < VRGDG_STENCIL_NONE || d->stencil_op > VRGDG_STENCIL_SOBEL_GPU) return fail(VRGDG_E_INVALID, "chain: bad stencil op %d", d->stencil_op);
  if (d->stencil_border != VRGDG_BORDER_REPLICATE && d->stencil_border != VRGDG_BORDER_ZERO) return fail(VRGDG_E_INVALID, "chain: bad border %d", d->stencil_border);
  if (d->post_grain_enabled && d->post_seed_mode != VRGDG_SEED_PER_CLIP && d->post_seed_mode != VRGDG_SEED_PER_FRAME) return fail(VRGDG_E_INVALID, "chain: bad post seed_mode");
  if ((int64_t)B * H * W == 0) return VRGDG_OK;
  LaunchCtx ctx;
  if ((rc = get_ctx(stream, ctx))) return rc;
  TileParams Q;
  memset(&Q, 0, sizeof(Q));
  Q.grid_limit = grid_limit;
  int mask = 0;
  bool exact = true;
  vrgdg_chain_desc dd = *d;
  if (cm_params) dd.cm_params = cm_params;
  dd.grain_frame0 += frame_offset;
  dd.post_frame0 += frame_offset;
  if ((rc = chain_point_params(&dd, B, H, W, Q.P, mask, exact, ext_noise, fast))) return rc;
  if (from_f) {
    if (dtype != VRGDG_F32 || !(mask & ST_CM)) return fail(VRGDG_E_INVALID, "chain: the f-plane pass needs fp32 frames and colour match");
    mask = (mask & ST_LUT) | ST_CMF;
    Q.P.ext_noise = nullptr;
  }
  const bool need_tile = dd.stencil_op != VRGDG_STENCIL_NONE || dd.post_grain_enabled;
  if (!need_tile) {
    if (mask == 0) {   // nothing enabled: copy
      if (in != out) {
        cudaError_t e = cudaMemcpyAsync(out, in, (size_t)B * H * W * 3 * elem_size(dtype), cudaMemcpyDeviceToDevice, ctx.stream);
        if (e != cudaSuccess) return fail_cuda(e, "chain copy");
      }
      return VRGDG_OK;
    }
#define PT(T) launch_point<T>(in, out, Q.P, mask, exact, ctx)
    cudaError_t e = DISPATCH_DTYPE(dtype, PT);
#undef PT
    if (e != cudaSuccess) return fail_cuda(e, "vrgdg_chain_apply");
    return VRGDG_OK;
  }
  Q.op = dd.stencil_op; Q.strength = dd.stencil_strength; Q.border = dd.stencil_border;
  Q.exact_stencil = (exact && (dtype == VRGDG_F32 || dtype == VRGDG_U8BGR)) ? 1 : 0;
  Q.post_enabled = dd.post_grain_enabled ? 1 : 0;
  Q.pI = dd.post_intensity; Q.ps = dd.post_sat; Q.poms = dd.post_one_minus_sat;
  Q.pseed = dd.post_seed; Q.pframe0 = dd.post_frame0; Q.pseed_mode = dd.post_seed_mode;
  grain_make_key(Q.pseed, Q.pseed_mode, Q.pkey);
  if (Q.post_enabled && mask == 0) mask = ST_POST;    // pure stencil + post grain: one Philox call per pixel pair via the grain plane
  return run_tile(in, out, B, H, W, dtype, Q, mask, exact, ctx);
}

static int chain_apply_impl(const void* in, void* out, int B, int H, int W, int dtype, const vrgdg_chain_desc* d,
                            const void* ext_noise, bool fast, void* stream) {
  return chain_apply_core(in, out, B, H, W, dtype, d, ext_noise, fast, stream, nullptr, false, 0);
}

int vrgdg_chain_apply(const void* in, void* out, int B, int H, int W, int dtype, const vrgdg_chain_desc* desc, void* stream) {
  return chain_apply_impl(in, out, B, H, W, dtype, desc, nullptr, false, stream);
}

/* same as vrgdg_chain_apply with the first grain stage reading N(0,1) from ext_noise ([B,H,W,3], frame dtype);
 * exists so that the fused chain can be compared bit-for-bit in arithmetic with the reference composition. */
int vrgdg_chain_apply_ext(const void* in, void* out, int B, int H, int W, int dtype, const vrgdg_chain_desc* desc,
                          const void* ext_noise, int flags, void* stream) {
  return chain_apply_impl(in, out, B, H, W, dtype, desc, ext_noise, (flags & VRGDG_CHAIN_FAST_MATH) != 0, stream);
}

static int chain_moments_impl(const void* in, int B, int H, int W, int dtype, const vrgdg_chain_desc* desc, const void* ext_noise,
                              double* sums, void* scratch, int64_t scratch_bytes, void* stream, const char* who) {
  if (!desc) return fail(VRGDG_E_INVALID, "%s: null descriptor", who);
  if (B < 0 || H <= 0 || W <= 0) return fail(VRGDG_E_INVALID, "%s: bad shape", who);
  PointParams P;
  zero_point(P, B, H, W);
  if (desc->grain_enabled) {
    if (desc->grain_seed_mode != VRGDG_SEED_PER_CLIP && desc->grain_seed_mode != VRGDG_SEED_PER_FRAME) return fail(VRGDG_E_INVALID, "%s: bad grain seed_mode %d", who, desc->grain_seed_mode);
    P.gI = desc->grain_intensity; P.gs = desc->grain_sat; P.goms = desc->grain_one_minus_sat;
    P.seed = desc->grain_seed; P.frame0 = desc->grain_frame0; P.seed_mode = desc->grain_seed_mode;
    grain_make_key(P.seed, P.seed_mode, P.gkey);
    P.ext_noise = ext_noise;
  }
  return moments_common(in, B, H, W, dtype, 0, H, desc->grain_enabled ? &P : nullptr, sums, scratch, scratch_bytes, stream, who);
}

int vrgdg_chain_lab_moments(const void* in, int B, int H, int W, int dtype, const vrgdg_chain_desc* desc, double* sums,
                            void* scratch, int64_t scratch_bytes, void* stream) {
  return chain_moments_impl(in, B, H, W, dtype, desc, nullptr, sums, scratch, scratch_bytes, stream, "vrgdg_chain_lab_moments");
}

/* same with the grain stage reading the external N(0,1) tensor of vrgdg_chain_apply_ext (exact arithmetic), so that the statistics
 * and the applied chain see the same grained frames */
int vrgdg_chain_lab_moments_ext(const void* in, int B, int H, int W, int dtype, const vrgdg_chain_desc* desc, const void* ext_noise,
                                double* sums, void* scratch, int64_t scratch_bytes, void* stream) {
  return chain_moments_impl(in, B, H, W, dtype, desc, ext_noise, sums, scratch, scratch_bytes, stream, "vrgdg_chain_lab_moments_ext");
}

/* ---- one call for a chain WITH colour match ------------------------------------------------------------------------------
 * scratch layout: [sums B x 7 doubles][params B x 12 floats, padded to 16 bytes][partials NB x G x 592 x 6 doubles]
 *                 [f-planes NB x G x H x W x 3 floats], NB = 2 buffers when the pipelined schedule can run (fp32 frames, more than
 *                 one group), else 1. */
static int cm_group_frames(int B, int H, int W, int dtype, int flags, int group_frames) {
  (void)dtype; (void)flags;
  if (group_frames > 0) return group_frames < B ? group_frames : (B > 0 ? B : 1);
  // Both passes are instruction-issue bound, so keeping a group's re-read set inside L2 (1-2 frames per group) buys nothing, while
  // short launches lose to their last partial wave of tiles.  Default = about
  // 64 Mpixel per group (8 x 4K, 32 x 1080p): > 25 000 tiles per launch, <= 800 MB of f-planes per buffer.
  const int64_t px = (int64_t)H * W;
  int64_t g = px > 0 ? (((int64_t)64 << 20) + px - 1) / px : 1;
  if (g < 1) g = 1;
  if (g > 64) g = 64;
  return g < B ? (int)g : (B > 0 ? B : 1);
}

static bool cm_wants_planes(int dtype, int flags) { return dtype == VRGDG_F32 && !(flags & VRGDG_CHAIN_CM_RECOMPUTE); }
static bool cm_uses_planes(int dtype, int H, int W, const void* in, int flags) {
  (void)H;
  return cm_wants_planes(dtype, flags) && (W % 4 == 0) && ((reinterpret_cast<uintptr_t>(in) & 15u) == 0);
}
static int cm_buffers(int B, int G, int dtype, int flags) {
  return (cm_wants_planes(dtype, flags) && !(flags & VRGDG_CHAIN_CM_SERIAL) && B > G) ? 2 : 1;
}

int64_t vrgdg_chain_cm_scratch_bytes(int B, int H, int W, int dtype, int flags, int group_frames) {
  if (B < 0 || H < 0 || W < 0 || !dtype_ok(dtype)) return 0;
  const int g = cm_group_frames(B, H, W, dtype, flags, group_frames);
  const int nb = cm_buffers(B, g, dtype, flags);
  int64_t n = (int64_t)B * 7 * 8;
  n += (((int64_t)B * 12 * 4 + 15) / 16) * 16;
  n += (int64_t)nb * g * MOMENT_BLOCKS * 6 * 8;
  if (cm_wants_planes(dtype, flags)) n += (int64_t)nb * ((((int64_t)g * H * W * 3 * 4) + 255) / 256) * 256;
  return n + 512;
}

/* Side streams of the pipelined schedule: one high- and one low-priority non-blocking stream per (thread, device), created on first
 * use and kept for the life of the thread (the library owns no other CUDA resources). */
struct CmStreams { cudaStream_t hi = nullptr, lo = nullptr; };
static int cm_streams(CmStreams*& out) {
  static thread_local CmStreams per_dev[64];
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return fail_cuda(e, "cudaGetDevice");
  if (dev < 0 || dev >= 64) return fail(VRGDG_E_UNSUPPORTED, "device index %d", dev);
  CmStreams& s = per_dev[dev];
  if (!s.hi) {
    int least = 0, greatest = 0;
    if ((e = cudaDeviceGetStreamPriorityRange(&least, &greatest)) != cudaSuccess) return fail_cuda(e, "cudaDeviceGetStreamPriorityRange");
    if ((e = cudaStreamCreateWithPriority(&s.hi, cudaStreamNonBlocking, greatest)) != cudaSuccess) return fail_cuda(e, "cudaStreamCreateWithPriority");
    if ((e = cudaStreamCreateWithPriority(&s.lo, cudaStreamNonBlocking, least)) != cudaSuccess) return fail_cuda(e, "cudaStreamCreateWithPriority");
  }
  out = &s;
  return VRGDG_OK;
}

int vrgdg_chain_cm_apply(const void* in, void* out, int B, int H, int W, int dtype, const vrgdg_chain_desc* desc,
                         const double* ref_sums, int n_ref, const void* ext_noise, int flags, void* scratch, int64_t scratch_bytes,
                         int group_frames, void* stream) {
  if (!desc) return fail(VRGDG_E_INVALID, "vrgdg_chain_cm_apply: null descriptor");
  if (!desc->colormatch_enabled) return fail(VRGDG_E_INVALID, "vrgdg_chain_cm_apply: the descriptor has no colour-match stage (use vrgdg_chain_apply)");
  int rc = check_frames(in, out, B, H, W, dtype, "vrgdg_chain_cm_apply");
  if (rc) return rc;
  if (n_ref != 1 && n_ref != B) return fail(VRGDG_E_INVALID, "vrgdg_chain_cm_apply: reference batch %d is neither 1 nor %d", n_ref, B);
  if (desc->grain_enabled && desc->grain_seed_mode != VRGDG_SEED_PER_CLIP && desc->grain_seed_mode != VRGDG_SEED_PER_FRAME)
    return fail(VRGDG_E_INVALID, "vrgdg_chain_cm_apply: bad grain seed_mode %d", desc->grain_seed_mode);
  if ((int64_t)B * H * W == 0) return VRGDG_OK;
  if (!ref_sums || !scratch) return fail(VRGDG_E_INVALID, "vrgdg_chain_cm_apply: null pointer");
  if (in == out) return fail(VRGDG_E_INVALID, "vrgdg_chain_cm_apply cannot run in place");
  if (reinterpret_cast<uintptr_t>(scratch) & 255u) return fail(VRGDG_E_ALIGN, "vrgdg_chain_cm_apply: scratch must be 256-byte aligned");
  if (scratch_bytes < vrgdg_chain_cm_scratch_bytes(B, H, W, dtype, flags, group_frames))
    return fail(VRGDG_E_INVALID, "vrgdg_chain_cm_apply: scratch too small (%lld < %lld)", (long long)scratch_bytes,
                (long long)vrgdg_chain_cm_scratch_bytes(B, H, W, dtype, flags, group_frames));
  LaunchCtx ctx;
  if ((rc = get_ctx(stream, ctx))) return rc;
  const int G = cm_group_frames(B, H, W, dtype, flags, group_frames);
  const bool planes = cm_uses_planes(dtype, H, W, in, flags);
  const int NB = cm_buffers(B, G, dtype, flags);
  // statistics pass of group g+1 beside the apply pass of group g: pays when the apply pass waits on the L1 data pipe (LUT gather) and
  // leaves issue slots free; a colour match without a LUT is instruction bound in BOTH passes and runs them one after the other
  const bool piped = planes && NB == 2 && desc->lut_enabled;
  char* sp = reinterpret_cast<char*>(scratch);
  double* sums = reinterpret_cast<double*>(sp);
  sp += (int64_t)B * 7 * 8;
  float* params = reinterpret_cast<float*>(sp);
  sp += (((int64_t)B * 12 * 4 + 15) / 16) * 16;
  double* partials[2] = {reinterpret_cast<double*>(sp), nullptr};
  sp += (int64_t)G * MOMENT_BLOCKS * 6 * 8;
  if (NB == 2) { partials[1] = reinterpret_cast<double*>(sp); sp += (int64_t)G * MOMENT_BLOCKS * 6 * 8; }
  sp = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(sp) + 255u) & ~(uintptr_t)255u);
  const int64_t plane_bytes = ((((int64_t)G * H * W * 3 * 4) + 255) / 256) * 256;
  float* fplanes[2] = {planes ? reinterpret_cast<float*>(sp) : nullptr, (planes && NB == 2) ? reinterpret_cast<float*>(sp + plane_bytes) : nullptr};
  const size_t es = elem_size(dtype);
  const size_t frame_bytes = (size_t)H * W * 3 * es;
  const size_t noise_es = (dtype == VRGDG_U8BGR) ? 4 : es;
  const bool fast = (flags & VRGDG_CHAIN_FAST_MATH) != 0;
  const int ngroups = (B + G - 1) / G;

  // Pipelined schedule (fp32 frames, several groups): the statistics pass (instruction-issue / XU bound, 128-thread blocks of 8 K
  // registers) of group g+1 runs on a low-priority side stream WHILE the apply pass (L1 data-pipe bound, two resident tile CTAs per
  // SM that leave exactly that much of the register file) of group g runs on a high-priority one; f-planes and partials are double
  // buffered; events fork the side streams from the caller's stream and join them back, so the call stays stream-ordered.
  // Tile CTAs of the apply pass while a statistics pass runs beside it: every tile CTA less frees registers for 3.5 more 128-thread
  // statistics blocks.  Default 0 = no limit; VRGDG_PIPE_TILE_CTAS overrides (tuning only).
  int tile_ctas = 0;
  if (piped) {
    const char* ev = getenv("VRGDG_PIPE_TILE_CTAS");
    tile_ctas = ev ? atoi(ev) : 0;
  }
  CmStreams* ss = nullptr;
  cudaEvent_t ev_start = nullptr, ev_p1[2] = {nullptr, nullptr}, ev_p2[2] = {nullptr, nullptr};
  LaunchCtx lo = ctx, hi = ctx;
  if (piped) {
    if ((rc = cm_streams(ss))) return rc;
    lo.stream = ss->lo; hi.stream = ss->hi;
    cudaError_t e = cudaEventCreateWithFlags(&ev_start, cudaEventDisableTiming);
    for (int i = 0; i < 2 && e == cudaSuccess; ++i) {
      e = cudaEventCreateWithFlags(&ev_p1[i], cudaEventDisableTiming);
      if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_p2[i], cudaEventDisableTiming);
    }
    if (e == cudaSuccess) e = cudaEventRecord(ev_start, ctx.stream);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(lo.stream, ev_start, 0);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(hi.stream, ev_start, 0);
    if (e != cudaSuccess) return fail_cuda(e, "vrgdg_chain_cm_apply (events)");
  }
  auto cleanup = [&]() {
    if (ev_start) cudaEventDestroy(ev_start);
    for (int i = 0; i < 2; ++i) { if (ev_p1[i]) cudaEventDestroy(ev_p1[i]); if (ev_p2[i]) cudaEventDestroy(ev_p2[i]); }
  };

  for (int gi = 0; gi < ngroups; ++gi) {
    const int g0 = gi * G, buf = piped ? (gi & 1) : 0;
    const int n = (B - g0 < G) ? B - g0 : G;
    const char* gin = reinterpret_cast<const char*>(in) + (size_t)g0 * frame_bytes;
    char* gout = reinterpret_cast<char*>(out) + (size_t)g0 * frame_bytes;
    const void* gnoise = ext_noise ? reinterpret_cast<const char*>(ext_noise) + (size_t)g0 * H * W * 3 * noise_es : nullptr;
    const LaunchCtx& c1 = piped ? lo : ctx;
    cudaError_t e = cudaSuccess;
    if (piped && gi >= 2) e = cudaStreamWaitEvent(lo.stream, ev_p2[buf], 0);      // the apply pass of group gi-2 has released this buffer
    if (e != cudaSuccess) { cleanup(); return fail_cuda(e, "vrgdg_chain_cm_apply (wait)"); }
    // pass 1: grain (recomputed from the counter-based generator or read from ext_noise) -> Lab statistics [+ f-planes]
    PointParams P;
    zero_point(P, n, H, W);
    if (desc->grain_enabled) {
      P.gI = desc->grain_intensity; P.gs = desc->grain_sat; P.goms = desc->grain_one_minus_sat;
      P.seed = desc->grain_seed; P.frame0 = desc->grain_frame0 + g0; P.seed_mode = desc->grain_seed_mode;
      grain_make_key(P.seed, P.seed_mode, P.gkey);
      P.ext_noise = gnoise;
    }
#define MO(T) launch_moments<T>(gin, P, desc->grain_enabled != 0, 0, H, sums + (int64_t)g0 * 7, partials[buf], c1, fplanes[buf], piped)
    e = DISPATCH_DTYPE(dtype, MO);
#undef MO
    if (e != cudaSuccess) { cleanup(); return fail_cuda(e, "vrgdg_chain_cm_apply (moments)"); }
    k_colormatch_params<<<(n + 127) / 128, 128, 0, c1.stream>>>(sums + (int64_t)g0 * 7, n, ref_sums + (n_ref == 1 ? 0 : (int64_t)g0 * 7), n_ref == 1 ? 1 : n,
                                                               params + (int64_t)g0 * 12);
    count_launch();
    if ((e = cudaGetLastError()) != cudaSuccess) { cleanup(); return fail_cuda(e, "vrgdg_chain_cm_apply (params)"); }
    if (piped) {
      if ((e = cudaEventRecord(ev_p1[buf], lo.stream)) == cudaSuccess) e = cudaStreamWaitEvent(hi.stream, ev_p1[buf], 0);
      if (e != cudaSuccess) { cleanup(); return fail_cuda(e, "vrgdg_chain_cm_apply (record)"); }
    }
    // pass 2: the fused apply, from the f-planes (no grain, no forward Lab) or from the frames
    rc = chain_apply_core(planes ? reinterpret_cast<const void*>(fplanes[buf]) : reinterpret_cast<const void*>(gin), gout, n, H, W, dtype, desc, gnoise, fast,
                          piped ? reinterpret_cast<void*>(hi.stream) : stream, params + (int64_t)g0 * 12, planes, g0, piped ? tile_ctas : 0);
    if (rc) { cleanup(); return rc; }
    if (piped) {
      if ((e = cudaEventRecord(ev_p2[buf], hi.stream)) != cudaSuccess) { cleanup(); return fail_cuda(e, "vrgdg_chain_cm_apply (record)"); }
    }
  }
  if (piped) {   // join: the caller's stream continues after the last apply pass (which follows every statistics pass)
    cudaError_t e = cudaStreamWaitEvent(ctx.stream, ev_p2[(ngroups - 1) & 1], 0);
    if (e == cudaSuccess && ngroups >= 2) e = cudaStreamWaitEvent(ctx.stream, ev_p2[(ngroups - 2) & 1], 0);
    cleanup();
    if (e != cudaSuccess) return fail_cuda(e, "vrgdg_chain_cm_apply (join)");
  }
  return VRGDG_OK;
}

int64_t vrgdg_adjust_scratch_bytes(int B, int H, int W, const vrgdg_adjust_desc* d) {
  if (!d || B < 0 || H < 0 || W < 0 || !d->enabled) return 0;
  const int n = (d->clarity_on ? 1 : 0) + (d->sharpen_on ? 1 : 0);
  return (int64_t)n * B * H * W * 3 * (int64_t)sizeof(float);
}

int vrgdg_adjust(const void* in, void* out, int B, int H, int W, int dtype, const vrgdg_adjust_desc* d, const float* xx,
                 const float* yy, void* scratch, int64_t scratch_bytes, void* stream) {
  if (!d) return fail(VRGDG_E_INVALID, "vrgdg_adjust: null descriptor");
  int rc = check_frames(in, out, B, H, W, dtype, "vrgdg_adjust");
  if (rc) return rc;
  if ((int64_t)B * H * W == 0) return VRGDG_OK;
  if (d->enabled && d->vignette_on && (!xx || !yy)) return fail(VRGDG_E_INVALID, "vrgdg_adjust: vignette needs the xx / yy ramps");
  if (d->enabled && d->clarity_on && (d->blur_kernel < 1 || d->blur_kernel > 9 || d->blur_kernel % 2 == 0 ||
                                      (d->blur_kernel >= 3 && (d->blur_kernel / 2 >= H || d->blur_kernel / 2 >= W))))
    return fail(VRGDG_E_INVALID, "vrgdg_adjust: blur kernel %d invalid for %d x %d frames", d->blur_kernel, H, W);
  const int64_t need = vrgdg_adjust_scratch_bytes(B, H, W, d);
  if (need > 0 && (!scratch || scratch_bytes < need)) return fail(VRGDG_E_INVALID, "vrgdg_adjust: scratch too small (%lld < %lld)", (long long)scratch_bytes, (long long)need);
  if (need > 0 && (reinterpret_cast<uintptr_t>(scratch) & 3u)) return fail(VRGDG_E_ALIGN, "vrgdg_adjust: scratch must be 4-byte aligned");
  LaunchCtx ctx;
  if ((rc = get_ctx(stream, ctx))) return rc;
  AdjustParams A;
  memset(&A, 0, sizeof(A));
  A.B = B; A.H = H; A.W = W;
  for (int i = 0; i < 3; ++i) A.off[i] = d->offset_rgb[i];
  A.exposure = d->exposure; A.contrast = d->contrast; A.saturation = d->saturation;
  A.hl = d->highlights; A.sh = d->shadows; A.wh = d->whites; A.bl = d->blacks;
  A.clarity_on = d->clarity_on; A.sharpen_on = d->sharpen_on; A.kbox = d->blur_kernel;
  A.clarity = d->clarity; A.sharpen = d->sharpen;
  A.fade_on = d->fade_on; A.vignette_on = d->vignette_on;
  A.fade_mul = d->fade_mul; A.fade_add = d->fade_add; A.vignette = d->vignette;
  A.xx = xx; A.yy = yy;
  float* s1 = reinterpret_cast<float*>(scratch);
  float* s2 = s1 ? s1 + (size_t)B * H * W * 3 : nullptr;
#define AJ(T) launch_adjust<T>(in, out, A, d->enabled ? 1 : 0, s1, s2, ctx)
  cudaError_t e = DISPATCH_DTYPE(dtype, AJ);
#undef AJ
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_adjust");
  return VRGDG_OK;
}

int vrgdg_resize(const void* in, void* out, int B, int Hs, int Ws, int channels, int Ht, int Wt, int dtype,
                 const vrgdg_resize_desc* d, void* stream) {
  if (!d) return fail(VRGDG_E_INVALID, "vrgdg_resize: null descriptor");
  if (!dtype_ok(dtype) || dtype == VRGDG_U8BGR) return fail(VRGDG_E_INVALID, "vrgdg_resize: float dtype expected, got %d", dtype);
  if (B < 0 || Hs < 0 || Ws < 0 || Ht < 0 || Wt < 0) return fail(VRGDG_E_INVALID, "vrgdg_resize: negative shape");
  if (channels != 3 && channels != 4) return fail(VRGDG_E_INVALID, "vrgdg_resize: channels must be 3 or 4, got %d", channels);
  if (d->mode < VRGDG_RESIZE_NEAREST || d->mode > VRGDG_RESIZE_AREA) return fail(VRGDG_E_INVALID, "vrgdg_resize: unknown mode %d", d->mode);
  if ((int64_t)B * Ht * Wt == 0) return VRGDG_OK;
  if (!in || !out) return fail(VRGDG_E_INVALID, "vrgdg_resize: null pointer");
  if (in == out) return fail(VRGDG_E_INVALID, "vrgdg_resize: in-place resampling is not supported");
  if (d->src_w < 1 || d->src_h < 1 || d->src_x0 < 0 || d->src_y0 < 0 || (int64_t)d->src_x0 + d->src_w > Ws ||
      (int64_t)d->src_y0 + d->src_h > Hs)
    return fail(VRGDG_E_INVALID, "vrgdg_resize: ROI %d,%d %dx%d outside %dx%d frames", d->src_x0, d->src_y0, d->src_w, d->src_h, Ws, Hs);
  if (d->res_w < 1 || d->res_h < 1) return fail(VRGDG_E_INVALID, "vrgdg_resize: resampled size %dx%d", d->res_w, d->res_h);
  LaunchCtx ctx;
  int rc = get_ctx(stream, ctx);
  if (rc) return rc;
  ResizeParams R;
  R.B = B; R.Hs = Hs; R.Ws = Ws; R.Cs = channels; R.Ht = Ht; R.Wt = Wt; R.mode = d->mode;
  R.x0 = d->src_x0; R.y0 = d->src_y0; R.sw = d->src_w; R.sh = d->src_h; R.rw = d->res_w; R.rh = d->res_h;
  R.ox = d->off_x; R.oy = d->off_y;
  R.scale_x = (float)d->src_w / (float)d->res_w;
  R.scale_y = (float)d->src_h / (float)d->res_h;
#define RZ(T) launch_resize<T>(in, out, R, ctx)
  cudaError_t e = (dtype == VRGDG_F32) ? RZ(float) : ((dtype == VRGDG_F16) ? RZ(__half) : RZ(__nv_bfloat16));
#undef RZ
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_resize");
  return VRGDG_OK;
}

int vrgdg_blend(const void* a, const void* b, void* out, int64_t n, int dtype, float weight_a, float weight_b, void* stream) {
  if (!dtype_ok(dtype) || dtype == VRGDG_U8BGR) return fail(VRGDG_E_INVALID, "vrgdg_blend: float dtype expected, got %d", dtype);
  if (n < 0) return fail(VRGDG_E_INVALID, "vrgdg_blend: negative element count");
  if (n == 0) return VRGDG_OK;
  if (!a || !b || !out) return fail(VRGDG_E_INVALID, "vrgdg_blend: null pointer");
  LaunchCtx ctx;
  int rc = get_ctx(stream, ctx);
  if (rc) return rc;
#define BL(T) launch_blend<T>(a, b, out, n, weight_a, weight_b, ctx)
  cudaError_t e = (dtype == VRGDG_F32) ? BL(float) : ((dtype == VRGDG_F16) ? BL(__half) : BL(__nv_bfloat16));
#undef BL
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_blend");
  return VRGDG_OK;
}

/* ---- histogram / CDF colour transfer (labelled extension, see vrgdg_histmatch.cuh) ---- */
int vrgdg_hist_counts(const void* in, int B, int H, int W, int dtype, int row0, int rows, uint32_t* counts, void* stream) {
  if (!dtype_ok(dtype)) return fail(VRGDG_E_INVALID, "vrgdg_hist_counts: unknown dtype %d", dtype);
  if (B < 0 || H <= 0 || W <= 0) return fail(VRGDG_E_INVALID, "vrgdg_hist_counts: bad shape [%d,%d,%d]", B, H, W);
  if (row0 < 0 || rows < 0 || row0 + rows > H) return fail(VRGDG_E_INVALID, "vrgdg_hist_counts: row range [%d,%d) outside [0,%d)", row0, row0 + rows, H);
  if ((int64_t)H * W >= (int64_t)1 << 31) return fail(VRGDG_E_UNSUPPORTED, "vrgdg_hist_counts: frame of %d x %d pixels exceeds 2^31 (32-bit counters)", H, W);
  if (B == 0) return VRGDG_OK;
  if (!in || !counts) return fail(VRGDG_E_INVALID, "vrgdg_hist_counts: null pointer");
  if (reinterpret_cast<uintptr_t>(counts) & 3u) return fail(VRGDG_E_ALIGN, "vrgdg_hist_counts: counts must be 4-byte aligned");
  LaunchCtx ctx;
  int rc = get_ctx(stream, ctx);
  if (rc) return rc;
#define HC(T) launch_hist_counts<T>(in, B, H, W, row0, rows, counts, ctx)
  cudaError_t e = DISPATCH_DTYPE(dtype, HC);
#undef HC
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_hist_counts");
  return VRGDG_OK;
}

int vrgdg_histmatch_tables(const uint32_t* frame_counts, int B, const uint32_t* ref_counts, int n_ref, float* tables, void* stream) {
  if (B < 0) return fail(VRGDG_E_INVALID, "vrgdg_histmatch_tables: negative B");
  if (B == 0) return VRGDG_OK;
  if (!frame_counts || !ref_counts || !tables) return fail(VRGDG_E_INVALID, "vrgdg_histmatch_tables: null pointer");
  if (n_ref != 1 && n_ref != B) return fail(VRGDG_E_INVALID, "vrgdg_histmatch_tables: reference batch %d is neither 1 nor %d", n_ref, B);
  if (reinterpret_cast<uintptr_t>(tables) & 7u) return fail(VRGDG_E_ALIGN, "vrgdg_histmatch_tables: tables must be 8-byte aligned");
  LaunchCtx ctx;
  int rc = get_ctx(stream, ctx);
  if (rc) return rc;
  k_hist_tables<<<B * 3, 256, 0, ctx.stream>>>(frame_counts, ref_counts, n_ref, reinterpret_cast<float2*>(tables));
  count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_histmatch_tables");
  return VRGDG_OK;
}

int vrgdg_histmatch_apply(const void* in, void* out, int B, int H, int W, int dtype, const float* tables, float t, float one_minus_t,
                          void* stream) {
  int rc = check_frames(in, out, B, H, W, dtype, "vrgdg_histmatch_apply");
  if (rc) return rc;
  if ((int64_t)B * H * W == 0) return VRGDG_OK;
  if (!tables) return fail(VRGDG_E_INVALID, "vrgdg_histmatch_apply: null tables");
  if (reinterpret_cast<uintptr_t>(tables) & 7u) return fail(VRGDG_E_ALIGN, "vrgdg_histmatch_apply: tables must be 8-byte aligned");
  LaunchCtx ctx;
  if ((rc = get_ctx(stream, ctx))) return rc;
#define HA(T) launch_histmatch_apply<T>(in, out, B, (int64_t)H * W, reinterpret_cast<const float2*>(tables), t, one_minus_t, ctx)
  cudaError_t e = DISPATCH_DTYPE(dtype, HA);
#undef HA
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_histmatch_apply");
  return VRGDG_OK;
}

int vrgdg_temporal_sharpen(const void* in, void* out, int B, int H, int W, int dtype, float strength, const void* prev_frame,
                           const void* next_frame, void* stream) {
  int rc = check_frames(in, out, B, H, W, dtype, "vrgdg_temporal_sharpen");
  if (rc) return rc;
  if ((int64_t)B * H * W == 0) return VRGDG_OK;
  const size_t es = elem_size(dtype);
  if ((prev_frame && reinterpret_cast<uintptr_t>(prev_frame) % es) || (next_frame && reinterpret_cast<uintptr_t>(next_frame) % es))
    return fail(VRGDG_E_ALIGN, "vrgdg_temporal_sharpen: halo frame pointer not aligned to its element size");
  if (in == out) return fail(VRGDG_E_INVALID, "vrgdg_temporal_sharpen cannot run in place (a frame is read again as its successor's neighbour)");
  LaunchCtx ctx;
  if ((rc = get_ctx(stream, ctx))) return rc;
  TemporalParams P;
  P.B = B; P.frame_elems = (int64_t)H * W * 3; P.strength = strength; P.prev = prev_frame; P.next = next_frame;
#define TS(T) launch_temporal<T>(in, out, P, ctx)
  cudaError_t e = DISPATCH_DTYPE(dtype, TS);
#undef TS
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_temporal_sharpen");
  return VRGDG_OK;
}

// OpenCV's interpolateLanczos4 (imgproc/resize.cpp), restated: note that x + 3 and x + 3 - i are FLOAT sums before the promotion
// to double, and the accumulation / normalisation of the eight weights is float as well
static void lanczos4_weights(float x, float* coeffs) {
  static const double s45 = 0.70710678118654752440084436210485;
  static const double cs[8][2] = {{1, 0}, {-s45, -s45}, {0, 1}, {s45, -s45}, {-1, 0}, {s45, s45}, {0, -1}, {-s45, s45}};
  const double pi = 3.1415926535897932384626433832795;
  float sum = 0.f;
  const float x3 = x + 3.f;
  const double y0 = (double)(-x3) * pi * 0.25, s0 = std::sin(y0), c0 = std::cos(y0);
  for (int i = 0; i < 8; ++i) {
    const float d = x3 - (float)i;
    if (std::fabs(d) >= 1e-6f) {
      const double y = (double)(-d) * pi * 0.25;
      coeffs[i] = (float)((cs[i][0] * s0 + cs[i][1] * c0) / (y * y));
    } else {
      coeffs[i] = 1e30f;                                   // the tap that sits exactly on a source sample takes all the weight
    }
    sum += coeffs[i];
  }
  sum = 1.f / sum;
  for (int i = 0; i < 8; ++i) coeffs[i] *= sum;
}

int vrgdg_lanczos4_tables(int src_size, int dst_size, int32_t* ofs, int16_t* coef) {
  if (src_size < 1 || dst_size < 1) return fail(VRGDG_E_INVALID, "vrgdg_lanczos4_tables: sizes %d -> %d", src_size, dst_size);
  if (!ofs || !coef) return fail(VRGDG_E_INVALID, "vrgdg_lanczos4_tables: null pointer");
  const double inv_scale = (double)dst_size / (double)src_size;
  const volatile double scale = 1.0 / inv_scale;            // cv::resize: scale_x = 1. / inv_scale_x (volatile: no fused multiply-add below)
  for (int d = 0; d < dst_size; ++d) {
    const volatile double prod = ((double)d + 0.5) * scale;
    float fx = (float)(prod - 0.5);
    const int sx = (int)std::floor(fx);
    fx -= (float)sx;
    ofs[d] = sx;
    float w[8];
    lanczos4_weights(fx, w);
    for (int k = 0; k < 8; ++k) {
      const long r = lrintf(w[k] * 2048.f);                  // saturate_cast<short>(cvRound(.)), round half to even
      coef[(size_t)d * 8 + k] = (int16_t)(r < -32768 ? -32768 : (r > 32767 ? 32767 : r));
    }
  }
  return VRGDG_OK;
}

int64_t vrgdg_lanczos4_scratch_bytes(int B, int Hs, int Wd) {
  if (B < 0 || Hs < 0 || Wd < 0) return 0;
  return (int64_t)B * Hs * Wd * 3 * (int64_t)sizeof(int32_t);
}

int vrgdg_lanczos4_resize_u8(const uint8_t* in, uint8_t* out, int B, int Hs, int Ws, int Hd, int Wd, const int32_t* xofs,
                             const int16_t* xcoef, const int32_t* yofs, const int16_t* ycoef, void* scratch, int64_t scratch_bytes,
                             void* stream) {
  if (B < 0 || Hs < 0 || Ws < 0 || Hd < 0 || Wd < 0) return fail(VRGDG_E_INVALID, "vrgdg_lanczos4_resize_u8: negative shape");
  if ((int64_t)B * Hd * Wd == 0) return VRGDG_OK;
  if (Hs < 1 || Ws < 1) return fail(VRGDG_E_INVALID, "vrgdg_lanczos4_resize_u8: empty source frames");
  if (!in || !out || !xofs || !xcoef || !yofs || !ycoef) return fail(VRGDG_E_INVALID, "vrgdg_lanczos4_resize_u8: null pointer");
  if (in == out) return fail(VRGDG_E_INVALID, "vrgdg_lanczos4_resize_u8: in-place resampling is not supported");
  if ((int64_t)Wd * 3 > 0x7FFFFFFF || (int64_t)Ws * 3 > 0x7FFFFFFF) return fail(VRGDG_E_UNSUPPORTED, "vrgdg_lanczos4_resize_u8: rows too long");
  const int64_t need = vrgdg_lanczos4_scratch_bytes(B, Hs, Wd);
  if (!scratch || scratch_bytes < need) return fail(VRGDG_E_INVALID, "vrgdg_lanczos4_resize_u8: scratch too small (%lld < %lld)", (long long)scratch_bytes, (long long)need);
  if ((reinterpret_cast<uintptr_t>(scratch) & 15u) || (reinterpret_cast<uintptr_t>(xcoef) & 15u) || (reinterpret_cast<uintptr_t>(ycoef) & 15u))
    return fail(VRGDG_E_ALIGN, "vrgdg_lanczos4_resize_u8: scratch and weight tables must be 16-byte aligned");
  if (((Wd * 3) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 3u)) return fail(VRGDG_E_ALIGN, "vrgdg_lanczos4_resize_u8: output must be 4-byte aligned");
  LaunchCtx ctx;
  int rc = get_ctx(stream, ctx);
  if (rc) return rc;
  LanczosParams L;
  L.B = B; L.Hs = Hs; L.Ws = Ws; L.Hd = Hd; L.Wd = Wd;
  L.xofs = xofs; L.xcoef = xcoef; L.yofs = yofs; L.ycoef = ycoef;
  cudaError_t e = launch_lanczos4(in, out, reinterpret_cast<int32_t*>(scratch), L, ctx);
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_lanczos4_resize_u8");
  return VRGDG_OK;
}

int vrgdg_u8bgr_to_rgb(const uint8_t* in, void* out, int64_t npix, int dtype, void* stream) {
  if (!dtype_ok(dtype) || dtype == VRGDG_U8BGR) return fail(VRGDG_E_INVALID, "vrgdg_u8bgr_to_rgb: float dtype expected, got %d", dtype);
  if (npix < 0) return fail(VRGDG_E_INVALID, "vrgdg_u8bgr_to_rgb: negative pixel count");
  if (npix == 0) return VRGDG_OK;
  if (!in || !out) return fail(VRGDG_E_INVALID, "vrgdg_u8bgr_to_rgb: null pointer");
  LaunchCtx ctx;
  int rc = get_ctx(stream, ctx);
  if (rc) return rc;
#define UI(T) launch_u8_in<T>(in, out, npix, ctx)
  cudaError_t e = (dtype == VRGDG_F32) ? UI(float) : ((dtype == VRGDG_F16) ? UI(__half) : UI(__nv_bfloat16));
#undef UI
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_u8bgr_to_rgb");
  return VRGDG_OK;
}

int vrgdg_rgb_to_u8bgr(const void* in, uint8_t* out, int64_t npix, int dtype, void* stream) {
  if (!dtype_ok(dtype) || dtype == VRGDG_U8BGR) return fail(VRGDG_E_INVALID, "vrgdg_rgb_to_u8bgr: float dtype expected, got %d", dtype);
  if (npix < 0) return fail(VRGDG_E_INVALID, "vrgdg_rgb_to_u8bgr: negative pixel count");
  if (npix == 0) return VRGDG_OK;
  if (!in || !out) return fail(VRGDG_E_INVALID, "vrgdg_rgb_to_u8bgr: null pointer");
  LaunchCtx ctx;
  int rc = get_ctx(stream, ctx);
  if (rc) return rc;
#define UO(T) launch_u8_out<T>(in, out, npix, ctx)
  cudaError_t e = (dtype == VRGDG_F32) ? UO(float) : ((dtype == VRGDG_F16) ? UO(__half) : UO(__nv_bfloat16));
#undef UO
  if (e != cudaSuccess) return fail_cuda(e, "vrgdg_rgb_to_u8bgr");
  return VRGDG_OK;
}

}  // extern "C"

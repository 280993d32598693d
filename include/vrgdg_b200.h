/*
 * vrgdg_b200.h — C ABI of libvrgdg_b200.so: H100 (sm_90a) kernels for the per-pixel video
 * post-processing hot path of the comfyui-vrgamedevgirl node pack.
 *
 * The reference is pure Python (no FFI of its own); each entry point below replaces the tensor
 * math of one reference function and is what a ctypes stub in the reference would bind
 * (see INTEGRATION.md).  Reference citations are file:line into the reference tree.
 *
 * Conventions
 *   - every function returns int: 0 = VRGDG_OK, <0 = VRGDG_E_*; text via vrgdg_last_error()
 *     (thread-local).  No C++ exceptions cross the boundary, no torch types in signatures.
 *   - all pointers are DEVICE pointers unless a name ends in _host; the library never allocates
 *     or frees frame memory (the caller's allocator owns it); `in` and `out` must not alias
 *     for the stencil / tile entry points.
 *   - frames are ComfyUI IMAGE layout [B,H,W,C] contiguous, channel fastest, values in [0,1].
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued there, nothing
 *     synchronises the device.  The current CUDA device must be the one owning the pointers.
 *   - dtype: element type of frames (and of ext_noise).  Arithmetic is fp32 inside the kernels.
 */
#ifndef VRGDG_B200_H
#define VRGDG_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VRGDG_ABI_VERSION 1

#if defined(__GNUC__)
#define VRGDG_API __attribute__((visibility("default")))
#else
#define VRGDG_API
#endif

enum {
  VRGDG_OK = 0,
  VRGDG_E_INVALID = -1,      /* bad argument (shape, enum, null pointer)  -> ValueError   */
  VRGDG_E_UNSUPPORTED = -2,  /* valid but not implemented combination      -> ValueError   */
  VRGDG_E_CUDA = -3,         /* CUDA runtime / driver error                -> RuntimeError */
  VRGDG_E_ALIGN = -4         /* pointer not aligned to the element size    -> ValueError   */
};

/* VRGDG_U8BGR: frames are uint8 in cv2's BGR order, the reference's video wire format (_frames_to_tensor / _tensor_to_frames,
 * VRGDG_LUTVideoTools.py:736-752): kernels read x/255.0, swap to RGB, compute in fp32 and write clip(y*255,0,255) truncated, BGR.
 * Accepted by vrgdg_grain, vrgdg_stencil3x3, vrgdg_lut3d_apply (3 channels), vrgdg_lab_moments, vrgdg_colormatch_apply and the
 * chain entry points: 6 bytes of HBM traffic per pixel instead of 24, no separate conversion passes.  ext_noise for uint8
 * frames is float32 [B,H,W,3] in RGB order. */
enum { VRGDG_F32 = 0, VRGDG_F16 = 1, VRGDG_BF16 = 2, VRGDG_U8BGR = 3 };

/* 3x3 stencil epilogues.  nodes.py:182-209 (box unsharp), :266-289 (laplacian, numpy path),
 * :249-258 (laplacian, torch path: opposite sign), :357-384 (sobel, numpy), :329-349 (sobel, torch: +1e-6) */
enum {
  VRGDG_STENCIL_NONE = 0,
  VRGDG_STENCIL_BOX_UNSHARP = 1,
  VRGDG_STENCIL_LAPLACIAN_CPU = 2,
  VRGDG_STENCIL_LAPLACIAN_GPU = 3,
  VRGDG_STENCIL_SOBEL_CPU = 4,
  VRGDG_STENCIL_SOBEL_GPU = 5
};

/* border of the 3x3 window: numpy paths use np.pad(mode="edge"); torch paths zero-pad. */
enum { VRGDG_BORDER_REPLICATE = 0, VRGDG_BORDER_ZERO = 1 };

/* how (seed, frame index) key the counter-based RNG.
 *   PER_CLIP : key = seed, counter carries the absolute frame index frame0+i
 *              (FastFilmGrain nodes.py:51, _apply_film_grain_tensor VRGDG_LUTVideoTools.py:268-272)
 *   PER_FRAME: key = (seed + frame0 + i) & 0x7FFFFFFF, frame counter = 0
 *              (_apply_seeded_grain VRGDG_StandaloneVideoEnhancerNodes.py:266-269)
 * Both make the result independent of batch boundaries and of how frames are sharded. */
enum { VRGDG_SEED_PER_CLIP = 0, VRGDG_SEED_PER_FRAME = 1 };
enum { VRGDG_RESIZE_NEAREST = 0, VRGDG_RESIZE_BILINEAR = 1, VRGDG_RESIZE_BICUBIC = 2, VRGDG_RESIZE_AREA = 3 };

/* ---- library ---------------------------------------------------------------------------- */
VRGDG_API int vrgdg_version(void);
VRGDG_API const char* vrgdg_last_error(void);
/* sm count and compute capability of the current device */
VRGDG_API int vrgdg_device_info(int* sm_count, int* cc_major, int* cc_minor);
/* number of kernel launches this library has enqueued since load (all threads) */
VRGDG_API int64_t vrgdg_launch_count(void);
/* name of the code path the last tile call on this thread took: "tma" or "generic" */
VRGDG_API const char* vrgdg_last_tile_path(void);

/* ---- 3D LUT, trilinear --------------------------------------------------------------------
 * Replaces VRGDG_LUTS._apply_cube_lut + the strength blend of apply_lut
 * (VRGDG_IV_Adjustments.py:289-343, :355-359; _apply_lut_tensor VRGDG_LUTVideoTools.py:172-185).
 * lut_packed: the table in the library's device layout, produced once per LUT by vrgdg_lut3d_pack from the
 * reference layout [S,S,S,3] fp32, index order [blue][green][red][rgb] (:272-274).  dmin/dspan_host: 3 floats
 * each on the HOST, dspan = clamp(dmax-dmin, 1e-6) already evaluated in the image dtype (:295,:351-352).
 * channels 3 or 4 (alpha copied through, :341-343).  blend in (0,1]: out = in*(1-blend)+lut*blend when
 * blend<1; one_minus_blend is passed separately because the reference forms (1.0-blend) in double.
 * Output is bit-identical to the reference CPU path for fp32 frames. */
VRGDG_API int64_t vrgdg_lut3d_packed_bytes(int lut_size);
/* lut: device [S,S,S,3] fp32 (reference layout); packed: device buffer of vrgdg_lut3d_packed_bytes(S), 32-byte aligned.
 * Entry (b,g,r) of the packed table = the 8 corners of the cell whose origin is (b,g,r) (neighbours clamped to S-1), 24 floats
 * = 96 bytes: a pixel's whole trilinear stencil arrives with three consecutive 32-byte sectors.  The buffer holds TWO tables of
 * S^3 x 96 bytes: the corner cells (every exact entry point: bit-identical lookups) followed by the same cells as coefficients
 * of the trilinear polynomial (differences of the corners formed in double, rounded once), which the chains that draw their own
 * grain evaluate with 7 FMAs per channel (fast arithmetic, a few 1e-8 of the table values away from the corner form). */
VRGDG_API int vrgdg_lut3d_pack(const float* lut, float* packed, int lut_size, void* stream);
VRGDG_API int vrgdg_lut3d_apply(const void* in, void* out, int64_t npix, int channels, int dtype,
                      const float* lut_packed, int lut_size,
                      const float* dmin_host, const float* dspan_host,
                      float blend, float one_minus_blend, void* stream);

/* ---- film grain ------------------------------------------------------------------------------
 * Replaces FastFilmGrain.apply_grain (nodes.py:49-60), _apply_film_grain_tensor
 * (VRGDG_LUTVideoTools.py:262-277) and _apply_seeded_grain (VRGDG_StandaloneVideoEnhancerNodes.py:261-275).
 * z ~ N(0,1) per element from Philox4x32-10 + Box-Muller keyed per seed_mode, or read from ext_noise
 * ([B,H,W,3], same dtype as frames) when non-null; then
 *   out = clamp(x + I*(sat*z' + one_minus_sat*z_g), 0, 1),  z' = (2 z_r, z_g, 3 z_b).
 * With ext_noise and fp32 frames every rounding step equals the reference's (bit-identical). */
VRGDG_API int vrgdg_grain(const void* in, void* out, int B, int H, int W, int dtype,
                float intensity, float sat, float one_minus_sat,
                uint64_t seed, int64_t frame0, int seed_mode,
                const void* ext_noise, void* stream);

/* ---- 3x3 stencil sharpeners --------------------------------------------------------------------
 * Replaces FastUnsharpSharpen / FastLaplacianSharpen / FastSobelSharpen (nodes.py:156-384) and
 * _apply_unsharp (VRGDG_StandaloneVideoEnhancerNodes.py:233-258).  TMA-tiled when rows are 16-byte
 * aligned, generic tile loader otherwise (same arithmetic). */
VRGDG_API int vrgdg_stencil3x3(const void* in, void* out, int B, int H, int W, int dtype,
                     int op, float strength, int border, void* stream);

/* ---- colour match (Reinhard LAB mean/std transfer) ---------------------------------------------
 * Replaces ColorMatchToReference.match_color (nodes.py:97-121) incl. kornia rgb_to_lab / lab_to_rgb.
 * Step 1: per-frame raw LAB sums over image rows [row0,row0+rows): sums[b] = {n, S_L, S_a, S_b, S_LL, S_aa, S_bb}
 *         (7 doubles per frame; fixed-order two-level reduction, deterministic).  Row ranges exist so the
 *         reference image can be sharded by rows across ranks and merged by addition.
 * Step 2: params[b] = {k[3] = sd_ref/sd_img, c0[3] = mu_ref - mu_img*k, mu_img[3], sd_img[3]} fp32, sd = unbiased std + 1e-5 (:99-100,:109-110);
 *         opaque to the caller, consumed by vrgdg_colormatch_apply / the chain.
 *         n_ref is 1 (broadcast) or B.
 * Step 3: out = clamp(lab_to_rgb(t*((lab-mu)/sd*sd_ref+mu_ref) + (1-t)*lab)). */
VRGDG_API int64_t vrgdg_lab_moments_scratch_bytes(int B);
VRGDG_API int vrgdg_lab_moments(const void* in, int B, int H, int W, int dtype, int row0, int rows,
                      double* sums, void* scratch, int64_t scratch_bytes, void* stream);
VRGDG_API int vrgdg_colormatch_params(const double* frame_sums, int B, const double* ref_sums, int n_ref,
                            float* params, void* stream);
VRGDG_API int vrgdg_colormatch_apply(const void* in, void* out, int B, int H, int W, int dtype,
                           const float* params, float t, float one_minus_t, void* stream);

/* ---- fused chain ---------------------------------------------------------------------------------
 * One pass over HBM for  grain -> colour match -> 3D LUT -> 3x3 stencil -> post-grain , any subset.
 * Composition semantics = the reference nodes applied one after another on fp32 tensors (each stage
 * clamps to [0,1] where its node clamps).  post_grain reproduces _apply_effects_batch
 * (VRGDG_StandaloneVideoEnhancerNodes.py:278-294: unsharp first, seeded grain second). */
typedef struct vrgdg_chain_desc {
  /* stage 1: grain before everything else */
  int32_t grain_enabled;
  float grain_intensity, grain_sat, grain_one_minus_sat;
  uint64_t grain_seed;
  int64_t grain_frame0;
  int32_t grain_seed_mode;
  /* stage 2: colour match with precomputed params [B][12] (device) */
  int32_t colormatch_enabled;
  const float* cm_params;
  float cm_t, cm_one_minus_t;
  /* stage 3: 3D LUT (packed table from vrgdg_lut3d_pack) */
  int32_t lut_enabled;
  const float* lut;
  int32_t lut_size;
  float lut_dmin[3], lut_dspan[3];
  float lut_blend, lut_one_minus_blend;
  /* stage 4: stencil */
  int32_t stencil_op;   /* VRGDG_STENCIL_* */
  float stencil_strength;
  int32_t stencil_border;
  /* stage 5: grain after the stencil */
  int32_t post_grain_enabled;
  float post_intensity, post_sat, post_one_minus_sat;
  uint64_t post_seed;
  int64_t post_frame0;
  int32_t post_seed_mode;
} vrgdg_chain_desc;

VRGDG_API int vrgdg_chain_apply(const void* in, void* out, int B, int H, int W, int dtype,
                      const vrgdg_chain_desc* desc, void* stream);

/* vrgdg_chain_apply with the first grain stage reading N(0,1) from ext_noise ([B,H,W,3], frame dtype) instead
 * of the in-kernel generator: lets the fused chain be compared with the reference composition on the same
 * noise tensor (nodes.py:51 draws it from torch's generator, which no CUDA kernel can reproduce). */
/* flags: VRGDG_CHAIN_FAST_MATH = run the arithmetic variant vrgdg_chain_apply uses when it draws its own noise (FMA-contracted
 * grain blend and LUT lerps) on the external noise, so that exactly the benchmarked code path can be compared with the
 * reference composition (<= 1e-5); 0 = one rounding per reference op (bit-exact stages). */
#define VRGDG_CHAIN_FAST_MATH 1
VRGDG_API int vrgdg_chain_apply_ext(const void* in, void* out, int B, int H, int W, int dtype,
                          const vrgdg_chain_desc* desc, const void* ext_noise, int flags, void* stream);

/* LAB sums of grain(x) (stage 1 of desc only) so that colour match can follow grain inside the chain
 * without materialising the grained frames. */
VRGDG_API int vrgdg_chain_lab_moments(const void* in, int B, int H, int W, int dtype,
                            const vrgdg_chain_desc* desc, double* sums,
                            void* scratch, int64_t scratch_bytes, void* stream);
/* vrgdg_chain_lab_moments for a chain run with vrgdg_chain_apply_ext: the grain stage reads the same external N(0,1) tensor
 * (null = the in-kernel generator), so the statistics describe exactly the frames the colour-match stage will see. */
VRGDG_API int vrgdg_chain_lab_moments_ext(const void* in, int B, int H, int W, int dtype,
                                const vrgdg_chain_desc* desc, const void* ext_noise, double* sums,
                                void* scratch, int64_t scratch_bytes, void* stream);

/* One call for a chain that contains the colour-match stage (desc->colormatch_enabled; desc->cm_params is ignored): per-frame
 * statistics of the colour-match input, parameters against ref_sums ([n_ref][7] doubles from vrgdg_lab_moments, n_ref 1 or B) and
 * the fused apply, scheduled in groups of frames (bounds the scratch; see group_frames).
 *   fp32 frames (default): pass 1 stores lab_f(XYZ/white) = (fx, fy, fz) of every pixel of the group in scratch ("f-planes",
 *     12 B/px); pass 2 starts from them, so the grain is drawn once and the forward Lab transform evaluated once per pixel
 *     (bit-identical to recomputing them: the stored values ARE the recomputed values).
 *   other dtypes, or flags & VRGDG_CHAIN_CM_RECOMPUTE: pass 2 re-reads the frames and recomputes grain + forward Lab.
 * group_frames: frames per group, 0 = about 64 Mpixel per group (8 x 4K, 32 x 1080p frames; at most 64): long enough launches
 *     that their last partial wave of tiles does not matter; small groups (1-2 frames) keep the f-planes inside L2 instead.
 * ext_noise / flags & VRGDG_CHAIN_FAST_MATH: as vrgdg_chain_apply_ext.  scratch: vrgdg_chain_cm_scratch_bytes() bytes of device
 * memory, 256-byte aligned, owned by the caller (contents undefined afterwards).  Must not run in place. */
#define VRGDG_CHAIN_CM_RECOMPUTE 2
/* VRGDG_CHAIN_CM_SERIAL: run the groups one after the other on the caller's stream.  Default for fp32 frames with more than one group:
 * the statistics pass of group g+1 overlaps the apply pass of group g (they saturate different pipes: instruction issue / XU vs the
 * L1 data pipe) on two internal side streams forked from and joined back to the caller's stream by events; f-planes double buffered.
 * Results are bit-identical either way. */
#define VRGDG_CHAIN_CM_SERIAL 4
VRGDG_API int64_t vrgdg_chain_cm_scratch_bytes(int B, int H, int W, int dtype, int flags, int group_frames);
VRGDG_API int vrgdg_chain_cm_apply(const void* in, void* out, int B, int H, int W, int dtype, const vrgdg_chain_desc* desc,
                         const double* ref_sums, int n_ref, const void* ext_noise, int flags,
                         void* scratch, int64_t scratch_bytes, int group_frames, void* stream);

/* ---- "adjust" pass of the Builder UI ---------------------------------------------------------------------------
 * Replaces _apply_adjust_tensor (VRGDG_LUTVideoTools.py:307-391): clamp, temperature/tint offset, exposure, contrast,
 * saturation, highlight/shadow/white/black masks, clarity (k x k reflect-padded box, k = min(9, odd(H), odd(W))), sharpen
 * (3 x 3 replicate-padded box), fade, vignette, clamp.  The descriptor carries the scalars exactly as the reference's Python
 * expressions produce them (the host mirror in video_tools.py evaluates those expressions in double and rounds to fp32 where
 * torch does); xx / yy are torch.linspace(-1, 1, W / H) on the device (only read when vignette_on).  Bit-identical to the
 * reference for fp32 frames.  scratch: vrgdg_adjust_scratch_bytes() bytes of device memory (0 when neither clarity nor
 * sharpen is on). */
typedef struct vrgdg_adjust_desc {
  int32_t enabled;
  float offset_rgb[3];                 /* temperature/400 - tint/900, tint/450, -temperature/400 - tint/900 */
  float exposure, contrast, saturation;/* 2**(e/100), 1 + c/100, 1 + s/100 */
  float highlights, shadows, whites, blacks;   /* h/220, s/220, w/240, b/240 */
  int32_t clarity_on, sharpen_on, blur_kernel;
  float clarity, sharpen;              /* c/100, s/100 */
  int32_t fade_on, vignette_on;
  float fade_mul, fade_add, vignette;  /* 1 - fade*0.35, fade*0.18, v/100 */
} vrgdg_adjust_desc;
VRGDG_API int64_t vrgdg_adjust_scratch_bytes(int B, int H, int W, const vrgdg_adjust_desc* desc);
VRGDG_API int vrgdg_adjust(const void* in, void* out, int B, int H, int W, int dtype, const vrgdg_adjust_desc* desc,
                 const float* xx, const float* yy, void* scratch, int64_t scratch_bytes, void* stream);

/* ---- resize / restore around the enhancer ----------------------------------------------------------
 * _resize_batch / _restore_batch (VRGDG_VideoEnhanceNodes.py:54-106): F.interpolate(mode, align_corners=False, size=...)
 * of an RGB ROI, then a crop ("Crop to fill"), zero letterbox bars ("Fit with letterbox") or nothing ("Stretch"), then
 * clamp(0,1).  The ROI [src_x0, src_x0+src_w) x [src_y0, src_y0+src_h) of in [B,Hs,Ws,channels] (channels 3 or 4, alpha
 * ignored) is resampled to res_w x res_h; output pixel (x, y) of out [B,Ht,Wt,3] is resampled pixel (x - off_x, y - off_y)
 * or 0 outside it.  Nearest and area are bit-identical to torch, bilinear / bicubic within fp32 rounding (2e-6). */
typedef struct vrgdg_resize_desc {
  int32_t mode;                          /* VRGDG_RESIZE_* */
  int32_t src_x0, src_y0, src_w, src_h;
  int32_t res_w, res_h;
  int32_t off_x, off_y;
} vrgdg_resize_desc;
VRGDG_API int vrgdg_resize(const void* in, void* out, int B, int Hs, int Ws, int channels, int Ht, int Wt, int dtype,
                 const vrgdg_resize_desc* desc, void* stream);
/* out = clamp(a * weight_a + b * weight_b, 0, 1), one rounding per operation: the restore blend
 * originals * (1 - strength) + restored * strength (VRGDG_VideoEnhanceNodes.py:408-414).  n = elements. */
VRGDG_API int vrgdg_blend(const void* a, const void* b, void* out, int64_t n, int dtype, float weight_a, float weight_b,
                void* stream);

/* ---- histogram / CDF colour transfer — LABELLED EXTENSION, no reference counterpart ---------------------------------------------
 * BASELINE.json's north_star and configs[2] describe colour match as a "two-pass per-channel histogram + monotone-CDF LUT mapping";
 * the reference's ColorMatchToReference is the LAB mean/std transfer above and holds no histogram (SURVEY D1).  This mode is
 * therefore specified here (csrc/vrgdg_histmatch.cuh has the formulas), parity "unpinned":
 *   vrgdg_hist_counts      per frame and RGB channel 256-bin counts over rows [row0,row0+rows) -> counts[B][3][256] uint32 (the call
 *                          zeroes them first; exact integers, so row-sharded reference counts from several ranks simply add)
 *   vrgdg_histmatch_tables per frame and channel the monotone map reference_CDF^-1(frame_CDF) at the 257 bin edges ->
 *                          tables[B][3][256][2] fp32 = {T[k], T[k+1]-T[k]}; n_ref = 1 (one reference for all frames) or B
 *   vrgdg_histmatch_apply  out = clamp(x*(1-t) + map(x)*t), map = piecewise-linear interpolation of T */
VRGDG_API int vrgdg_hist_counts(const void* in, int B, int H, int W, int dtype, int row0, int rows, uint32_t* counts, void* stream);
VRGDG_API int vrgdg_histmatch_tables(const uint32_t* frame_counts, int B, const uint32_t* ref_counts, int n_ref, float* tables, void* stream);
VRGDG_API int vrgdg_histmatch_apply(const void* in, void* out, int B, int H, int W, int dtype, const float* tables,
                          float t, float one_minus_t, void* stream);

/* ---- temporal 3-frame unsharp (BASELINE.json configs[4]) — LABELLED EXTENSION, no reference counterpart --------------------
 * The reference has no temporal operator (VRGDG_VideoEnhanceNodes.py holds no sharpen / blur / stencil; SURVEY D4), so the
 * specification is this library's:  out[t] = clamp(x[t] + s * (x[t] - (x[t-1] + x[t] + x[t+1]) / 3), 0, 1), fp32, one rounding
 * per operation in that order, frames outside the clip replicated.  prev_frame / next_frame: the frame before in[0] / after
 * in[B-1] when the clip is sharded across calls or ranks (device pointers, one frame each, frame dtype), or null at the clip's
 * ends.  Must not run in place. */
VRGDG_API int vrgdg_temporal_sharpen(const void* in, void* out, int B, int H, int W, int dtype, float strength,
                           const void* prev_frame, const void* next_frame, void* stream);

/* ---- Lanczos4 resize of uint8 frames -----------------------------------------------------------------
 * _resize_frames (VRGDG_StandaloneVideoEnhancerNodes.py:213-230) = cv2.resize(frame, (w, h), interpolation=cv2.INTER_LANCZOS4)
 * on uint8 HWC frames; bit-identical to OpenCV 4.x (fixed-point 8-tap tables, border replication).
 * vrgdg_lanczos4_tables is HOST code (no device work): for one axis it fills ofs[dst_size] (source index of the 4th tap) and
 * coef[dst_size * 8] (weights x 2048 as shorts) exactly as OpenCV builds them; the caller uploads both axes' tables (coef
 * 16-byte aligned) and passes device pointers.  scratch: vrgdg_lanczos4_scratch_bytes() of device memory, 16-byte aligned
 * (the int32 horizontal pass).  in [B,Hs,Ws,3] u8 -> out [B,Hd,Wd,3] u8, channel order untouched. */
VRGDG_API int vrgdg_lanczos4_tables(int src_size, int dst_size, int32_t* ofs, int16_t* coef);
VRGDG_API int64_t vrgdg_lanczos4_scratch_bytes(int B, int Hs, int Wd);
VRGDG_API int vrgdg_lanczos4_resize_u8(const uint8_t* in, uint8_t* out, int B, int Hs, int Ws, int Hd, int Wd,
                             const int32_t* xofs, const int16_t* xcoef, const int32_t* yofs, const int16_t* ycoef,
                             void* scratch, int64_t scratch_bytes, void* stream);

/* ---- uint8 BGR wire format -------------------------------------------------------------------------
 * _frames_to_tensor / _tensor_to_frames (VRGDG_LUTVideoTools.py:736-752,
 * VRGDG_StandaloneVideoEnhancerNodes.py:311-324): u8 BGR -> RGB float /255.0 and
 * clip(x*255,0,255) truncated to u8 -> BGR. */
VRGDG_API int vrgdg_u8bgr_to_rgb(const uint8_t* in, void* out, int64_t npix, int dtype, void* stream);
VRGDG_API int vrgdg_rgb_to_u8bgr(const void* in, uint8_t* out, int64_t npix, int dtype, void* stream);

/* Raw N(0,1) stream of the grain generator ([B,H,W,3] fp32), for distribution tests. */
VRGDG_API int vrgdg_grain_noise(float* out, int B, int H, int W, uint64_t seed, int64_t frame0,
                      int seed_mode, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VRGDG_B200_H */

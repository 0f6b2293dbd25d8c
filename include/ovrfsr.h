/*
 * ovrfsr.h -- C ABI of the H100-native FSR1 / NIS eye-texture post-process.
 *
 * This is the drop-in boundary for ONE path of fholger/openvr_fsr: the per-eye pass that
 * vr::PostProcessor::Apply runs from the IVRCompositor::Submit hook
 * (src/postprocess/PostProcessor.cpp:123-164, called from src/postprocess/VrHooks.cpp:53,71,84).
 * Everything D3D11 did on that path (compute-shader dispatch of fsr_easu / fsr_rcas /
 * NIS_Upscale / NIS_Sharpen, constant buffers, intermediate textures) is behind these calls
 * as hand-written sm_90a CUDA kernels.  Plain pointers and sizes only; no C++ or torch
 * types cross this boundary.  All citations are relative to /root/reference/.
 *
 * The C++ class a maintainer links instead of the D3D11 one is
 * openvr_fsr_b200/csrc/postprocessor.h (same Apply/Reset surface); INTEGRATION.md shows
 * the binding.  There is NO CPU fallback: every entry point that launches work returns
 * OVRFSR_ERR_CUDA if no sm_90 device / driver is usable.
 */
#ifndef OVRFSR_H
#define OVRFSR_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define OVRFSR_API __declspec(dllexport)
#else
#define OVRFSR_API __attribute__((visibility("default")))
#endif

#define OVRFSR_VERSION 0x00010000u

/* status codes.  The reference's error convention is "log, disable, pass the frame through"
 * (PostProcessor.cpp:23-28,145-152); the C++ wrapper maps any non-zero status to that. */
typedef enum ovrfsr_status {
  OVRFSR_OK = 0,
  OVRFSR_ERR_INVALID = 1,     /* null / malformed argument */
  OVRFSR_ERR_UNSUPPORTED = 2, /* format or scale the path does not handle */
  OVRFSR_ERR_CUDA = 3,        /* CUDA runtime / driver failure, or no device */
  OVRFSR_ERR_NOMEM = 4,
  OVRFSR_PASSTHROUGH = 5      /* fsr_enabled == 0: nothing done, caller submits its own texture */
} ovrfsr_status;

/* pixel formats: the DXGI formats the path binds (PostProcessor.cpp:30-74) */
typedef enum ovrfsr_format {
  OVRFSR_FORMAT_RGBA8 = 0,   /* DXGI_FORMAT_R8G8B8A8_UNORM (sRGB variants are viewed as UNORM, :50-61) */
  OVRFSR_FORMAT_BGRA8 = 1,   /* DXGI_FORMAT_B8G8R8A8_UNORM */
  OVRFSR_FORMAT_RGBA16F = 2, /* DXGI_FORMAT_R16G16B16A16_FLOAT */
  OVRFSR_FORMAT_RGBA32F = 3, /* DXGI_FORMAT_R32G32B32A32_FLOAT (input: PostProcessor.cpp:32-33; as an output it
                                exposes the pre-quantisation result) */
  OVRFSR_FORMAT_RGB10A2 = 4, /* DXGI_FORMAT_R10G10B10A2_UNORM: one little-endian u32 per texel, R bits 0-9, G 10-19,
                                B 20-29, A 30-31.  As an output it is only produced from an RGB10A2 source -- the case
                                DetermineOutputFormat() exists for (:63-74) */
  OVRFSR_FORMAT_BGRX8 = 5,   /* DXGI_FORMAT_B8G8R8X8_UNORM (:54-55): source only; the X byte reads as alpha 1 */
  OVRFSR_FORMAT_RGB32F = 6,  /* DXGI_FORMAT_R32G32B32_FLOAT (:34-35): source only, 12 bytes per texel, alpha reads as 1;
                                ovrfsr_apply expands it to RGBA32F first (ovrfsr_expand_rgb32f), the stateless dispatches
                                return OVRFSR_ERR_UNSUPPORTED for it */
  OVRFSR_FORMAT_AUTO = -1    /* output only: DetermineOutputFormat(), :63-74 -> RGB10A2 for an RGB10A2 source, else RGBA8 */
} ovrfsr_format;

/* DXGI variant tags, OR-ed into ovrfsr_image::format of a SOURCE image.  The kernels view _SRGB and _TYPELESS textures as
 * plain UNORM (MakeSrgbFormatsTypeless / TranslateTypelessFormats, PostProcessor.cpp:30-61: no sRGB decode happens on this
 * path), so the tags change no pixel; they exist so that vr::PostProcessor can reproduce the colour-space tag the
 * reference hands to the real Submit (inputIsSrgb, :504 with IsConsideredSrgbByOpenVR, :76-92). */
#define OVRFSR_FORMAT_LAYOUT_MASK 0xff
#define OVRFSR_FORMAT_SRGB_BIT 0x100     /* DXGI_FORMAT_*_UNORM_SRGB */
#define OVRFSR_FORMAT_TYPELESS_BIT 0x200 /* DXGI_FORMAT_*_TYPELESS */
/* Storage tag, OR-ed into ovrfsr_image::format of a source or destination: `data` is a cudaArray_t (block-linear, e.g.
 * level 0 of the cudaMipmappedArray_t that cudaExternalMemoryGetMappedMipmappedArray returns for an imported Vulkan /
 * D3D12 texture, via cudaGetMipmappedArrayLevel), `pitch` and `slice_pitch` are ignored, and array_slices > 1 means a
 * layered array (cudaArrayLayered) whose layer 1 holds the right eye.  The array's channel descriptor must be the RAW one
 * of the format -- RGBA8 / BGRA8 / BGRX8: 4 x 8-bit cudaChannelFormatKindUnsigned; RGB10A2: 1 x 32-bit Unsigned;
 * RGBA16F: 4 x 16-bit Float; RGBA32F: 4 x 32-bit Float -- because the UnsignedNormalized kinds would decode in the
 * texture unit, bypassing the exact UNORM decodes strict math relies on; a binding chooses the descriptor when it maps
 * the memory.  Checked with cudaArrayGetInfo before anything is launched:
 *   OVRFSR_ERR_INVALID      unknown handle, or an extent / layer count other than width x height x array_slices
 *   OVRFSR_ERR_UNSUPPORTED  another channel descriptor, RGB32F (CUDA has no 3-component arrays), sample_count > 1, and
 *                           for a destination: a layered array or one without cudaArraySurfaceLoadStore
 * Accepted by ovrfsr_apply / _apply_pair (source), ovrfsr_apply_into / _apply_pair_into (source and destination),
 * ovrfsr_dispatch_fsr_easu / _fsr_rcas / _nis_scaler / _nis_sharpen (source and destination) and ovrfsr_image_copy.
 * ovrfsr_dispatch_fsr_fused, ovrfsr_dispatch_cas, ovrfsr_resolve_msaa and ovrfsr_expand_rgb32f return
 * OVRFSR_ERR_UNSUPPORTED for an array image, and OVRFSR_FLAG_FUSED_FSR falls back to the two dispatches for one.
 * The library reads and writes an array through texture / surface objects it creates on first use and keeps: call
 * ovrfsr_release_array before cudaFreeArray / cudaFreeMipmappedArray / cudaDestroyExternalMemory on any array passed in. */
#define OVRFSR_FORMAT_ARRAY_BIT 0x400

/* arithmetic mode of the kernels */
typedef enum ovrfsr_math {
  OVRFSR_MATH_FAST = 0,  /* FMA contraction + regrouped taps: each pass is <= 1 LSB (RGBA8) from the reference lines
                            on identical inputs.  Note that EASU -> RGBA8 -> RCAS amplifies a 1-LSB intermediate
                            difference in dark regions (RCAS divides by the ring maximum), as it does between any two
                            D3D11 GPUs; use STRICT when the composed result must match to the bit.  Measured on the
                            C2-sized test images: max 3 LSB, < 6e-6 of the channel values beyond 1 LSB (asserted <= 4
                            LSB / 1e-4 in tests/test_gpu_fsr_parity.py). */
  OVRFSR_MATH_STRICT = 1 /* the reference's operation order, no contraction: bit-identical to the reference lines,
                            end to end.  The default of ovrfsr_config_default. */
} ovrfsr_math;

/* Device-resident image: the CUDA analogue of the ID3D11Texture2D* that Texture_t::handle
 * carries (headers/openvr.h:177-182).  data is a device pointer unless stated otherwise (OVRFSR_FORMAT_ARRAY_BIT). */
typedef struct ovrfsr_image {
  void *data;
  uint32_t width;
  uint32_t height;
  uint32_t pitch;       /* bytes per row; rows need not be tightly packed */
  int32_t format;       /* ovrfsr_format */
  uint32_t array_slices;/* >1: right eye lives in slice 1 (PostProcessor.cpp:254-268); 0 is treated as 1 */
  uint32_t slice_pitch; /* bytes between slices when array_slices > 1 */
  uint32_t sample_count;/* >1: multisampled source (D3D11_TEXTURE2D_DESC::SampleDesc.Count): the samples of one texel
                           are consecutive, row = width*sample_count texel-sized entries; ovrfsr_apply resolves it
                           first like GetInputView's ResolveSubresource (PostProcessor.cpp:219-226).  0 = 1. */
} ovrfsr_image;

/* The Config fields that steer the path (src/postprocess/Config.h:11-17) plus what the
 * reference pulls from the live runtime (projection centres, PostProcessor.cpp:104-121). */
typedef struct ovrfsr_config {
  uint32_t struct_size;   /* sizeof(ovrfsr_config) */
  int32_t fsr_enabled;    /* Config::fsrEnabled */
  int32_t use_nis;        /* Config::useNis */
  float render_scale;     /* Config::renderScale */
  float sharpness;        /* Config::sharpness */
  float radius;           /* Config::radius */
  int32_t debug_mode;     /* Config::debugMode: tints the outside-radius region, enables timing */
  float proj_centre[4];   /* {leftX,leftY,rightX,rightY}; 0.5 each for a symmetric HMD */
  int32_t device;         /* CUDA device ordinal, -1 = current device */
  int32_t output_format;  /* ovrfsr_format, AUTO = reference behaviour */
  int32_t math_mode;      /* ovrfsr_math */
  int32_t flags;          /* OVRFSR_FLAG_* bits; 0 = defaults */
  int32_t reserved[4];
} ovrfsr_config;

/* ovrfsr_config::flags */
/* Run EASU -> RCAS as ONE fused kernel that keeps the upscaled image in shared memory (same output bits, 79.7 -> 35.0 MB
 * of traffic per C2 eye, one launch) whenever both passes run on the FSR path and the intermediate is UNORM (RGBA8 /
 * RGB10A2).  Off by default: the pass is instruction-issue-bound, not traffic-bound, and the fused kernel's
 * recomputed ring and lower occupancy make it slower than the two dispatches (DESIGN.md section 5).  Default (bit clear): the reference's two dispatches (PostProcessor.cpp:586-594),
 * with the outside-radius pixels written straight to the final image by the first one. */
#define OVRFSR_FLAG_FUSED_FSR 1
/* HDR float eye textures through AMD's simple reversible tone mapper (ffx_fsr1.h: FsrSrtmF / FsrSrtmInvF), an extension
 * the reference never enables.  EASU's luma analysis and RCAS's limiter assume display-referred values in [0, 1]; with
 * linear HDR input (scRGB, highlights above 1) the limiter's bound hitMax = (1 - mx) / (4 mn - 4) no longer prevents
 * overshoot.  With this bit the FSR passes run on
 *   F(c) = c / (max3(c.rgb) + 1)                      [0, 65504] -> [0, 0.9999848]
 * and the last one maps its result back with
 *   G(c) = c / max(1/32768, 1 - max3(c.rgb))          so G(c) <= 32768 x max3(c.rgb): the peak is 32768
 * (alpha untouched, IEEE reciprocal in both math modes).  It takes effect on the FSR path with a float source (RGBA16F,
 * RGBA32F, RGB32F after its expansion, a multisampled one after its resolve) and is ignored -- same output bits as with
 * the bit clear -- for UNORM sources and for use_nis.  With both passes the intermediate is RGBA32F for a float output
 * and RGBA16F for a UNORM output (an FP16 tone-mapped value near 1 is too coarse for HDR output once G amplifies it,
 * irrelevant where the output clips at 1; DESIGN.md section 4); the pairing and OVRFSR_FLAG_FUSED_FSR do not apply.  With
 * RCAS alone the outside-radius copy also runs in tone-mapped space (G(tint x F(c))): close to a copy, not bit-exact.
 * Negative, NaN and infinite channels are outside the tone map's domain: they go through the same formula and get
 * whatever IEEE arithmetic gives (e.g. max3 = -1 divides by zero).  Changing the bit through ovrfsr_set_config resets
 * the ctx like any config change. */
#define OVRFSR_FLAG_SRTM 2
/* The same tone map around the NIS pass (NVScaler or NVSharpen), an extension the reference never enables.
 * NVScalerUpdateConfig tunes the edge threshold kDetectThres, the contrast ratios and the sharpening strengths and
 * limits kSharpStrength* / kSharpLimit* for luma in [0, 1]; the passes then add a luma correction to the bilinear
 * colour, and above 1 the limiter no longer limits, so linear HDR highlights ring.  With this bit, on the NIS path with a
 * float source (RGBA16F, RGBA32F, RGB32F after its expansion, a multisampled one after its resolve), F is applied to
 * every source texel right after its decode and G to every stored pixel right before its encode: the pass filters
 * F(source), and outside the radius the copy is G(tint x bilinear(F(texels))), close to a copy but not bit-exact.  Same
 * maps, same arithmetic and same out-of-domain behaviour as OVRFSR_FLAG_SRTM; alpha untouched.  A NIS pass is a single
 * pass, so there is no intermediate: the output keeps the ctx's output format.  Ignored -- same output bits as with the
 * bit clear -- for UNORM sources and on the FSR path.  OVRFSR_FLAG_SRTM keeps its meaning and is still ignored on NIS;
 * a config with both bits tone-maps whichever path runs (a host with a use_nis toggle).  This is not the NIS SDK's
 * NIS_HDR_MODE_LINEAR / _PQ.  Changing the bit through ovrfsr_set_config resets the ctx like any config change. */
#define OVRFSR_FLAG_SRTM_NIS 4
/* Keep infinities and NaNs of float eye textures out of every pass and every stored pixel, an extension the reference
 * never enables.  An R16G16B16A16_FLOAT render target overflows to +-inf at 65520, one bad shader pixel can be NaN, and
 * the filters multiply every texel they read by its weight (inf x 0 = NaN), so one such texel can blacken a UNORM
 * output pixel or reach the compositor as NaN in a float one.  With this bit, on the FSR and NIS paths with a float
 * source (RGBA16F, RGBA32F, RGB32F after its expansion, a multisampled one after its resolve):
 *   finite-in   every channel of every texel a pass decodes: NaN -> +0, +-inf -> +-65504 (the largest RGBA16F value);
 *               every finite value is kept bit for bit, FP32 values beyond 65504 included.  Before F of the tone map.
 *   finite-out  every channel of every pixel a pass stores into a float image, the ctx's intermediate included:
 *               NaN -> +0, clamped to +-65504 (RGBA16F, then rounded) or +-FLT_MAX (RGBA32F).  After G of the tone map.
 * UNORM stores are unchanged (saturate already maps NaN to 0).  The passes, the intermediate's format, the pairing and
 * OVRFSR_FLAG_FUSED_FSR are exactly those of the bit clear; the MSAA resolve and the RGB32F expansion are not changed.
 * Ignored -- same output bits as with the bit clear -- for UNORM sources; on content without infinities or NaNs whose
 * outputs fit the destination it gives the bits of the bit clear too.  Not a repair: a bad texel still weighs in as 0 or
 * 65504, not as its neighbours.  Changing the bit through ovrfsr_set_config resets the ctx like any config change. */
#define OVRFSR_FLAG_FINITE 8
/* Filter linear float eye textures in a perceptual space, and store 8-bit outputs sRGB-encoded, an extension the
 * reference never enables.  EASU's edge analysis, RCAS's limiter and the NIS thresholds and limits are tuned for
 * gamma-encoded values, which the reference only feeds them for an 8-bit sRGB eye; and a linear value stored as plain
 * UNORM8 reads as dark and banded where the compositor takes the 8-bit output as sRGB.  With this bit, on the FSR and
 * NIS paths with a float source (RGBA16F, RGBA32F, RGB32F after its expansion, a multisampled one after its resolve):
 *   perceptual-in   every texel a pass decodes, after finite-in and F of the tone map: P(c) = copysign(sqrt(|c|), c)
 *                   on R, G and B (gamma 2.0, extended to negative channels by sign).
 *   perceptual-out  every pixel a pass stores, before G of the tone map: c * |c| on R, G and B.  A UNORM8 store then
 *                   sRGB-encodes the linear value v: code(v) = the number of k in 1..255 with v >= T[k], T[k] the
 *                   smallest binary32 at or above srgb_to_linear((k - 0.5) / 255) (D3D11's FLOAT -> SRGB conversion
 *                   without its 0.6-ulp slack; NaN and v <= 0 give 0).  Float stores keep the linear value.
 * Alpha is untouched.  sqrt and the product are correctly rounded in both math modes, so the maps are bit-exact.
 * FSR runs without the pairing and OVRFSR_FLAG_FUSED_FSR: EASU stores perceptual values into an RGBA16F intermediate
 * (RGBA32F for a float output) and RCAS maps them back; RCAS alone runs both maps, and so does the NIS pass.  The
 * outside-radius copies become encode(G(P^-1(tint x P(F(c))))): close to a copy, not bit-exact.  When the last pass
 * sRGB-encodes (an RGBA8 output), the image ovrfsr_apply / ovrfsr_apply_pair return carries OVRFSR_FORMAT_SRGB_BIT,
 * and ovrfsr_apply_into / _pair_into accept a destination of the output format with or without that tag.  Negative,
 * NaN and infinite channels get whatever IEEE arithmetic gives (OVRFSR_FLAG_FINITE keeps the last two out).  Ignored --
 * same output bits as with the bit clear -- for UNORM sources.  Changing the bit through ovrfsr_set_config resets the
 * ctx like any config change. */
#define OVRFSR_FLAG_PERCEPTUAL 16

typedef struct ovrfsr_ctx ovrfsr_ctx;

/* ---- lifetime ------------------------------------------------------------------------- */
/* Fills cfg with the reference defaults (Config.h:11-17: enabled=false, renderScale=1,
 * sharpness=0.75, radius=0.5) and proj centres 0.5. */
OVRFSR_API void ovrfsr_config_default(ovrfsr_config *cfg);
/* Replaces the `PostProcessor postProcessor;` global (VrHooks.cpp:19).  No GPU work happens here. */
OVRFSR_API int ovrfsr_create(ovrfsr_ctx **out, const ovrfsr_config *cfg);
OVRFSR_API void ovrfsr_destroy(ovrfsr_ctx *ctx);
/* PostProcessor::Reset (PostProcessor.cpp:166-194): drops every cached resource, re-enables. */
OVRFSR_API int ovrfsr_reset(ovrfsr_ctx *ctx);
/* What the hotkeys do (PostProcessor.cpp:670-704): mutate Config, then Reset -- on any change, sharpness included.
 * A host that changes the sharpness while the game runs calls ovrfsr_set_sharpness instead, which needs no reset. */
OVRFSR_API int ovrfsr_set_config(ovrfsr_ctx *ctx, const ovrfsr_config *cfg);
OVRFSR_API int ovrfsr_get_config(const ovrfsr_ctx *ctx, ovrfsr_config *cfg);

/* ---- the hot path --------------------------------------------------------------------- */
/* PostProcessor::Apply minus the OpenVR types (PostProcessor.cpp:123-164,563-638).
 *   eye           EVREye (0 left, 1 right)
 *   src           borrowed, read-only
 *   only_one_eye  |uMax-uMin| > .5 of the submit bounds (:146); 0 = both eyes side by side in src
 *   out           receives the ctx-owned output image (upscaled+sharpened); valid until the next
 *                 apply for the same eye, reset or destroy.  One output per eye (the reference
 *                 shares one between both eyes, PostProcessor.h:43,58).  Its format carries
 *                 OVRFSR_FORMAT_SRGB_BIT when the output is sRGB-encoded (OVRFSR_FLAG_PERCEPTUAL); it can be passed
 *                 back as a source as it is, but a host that passes it as a destination (ovrfsr_image_copy, a
 *                 dispatch) clears the tag first.
 *   stream        cudaStream_t; work is enqueued asynchronously, nothing is synchronised.  The ctx reuses its per-eye
 *                 intermediates and outputs on every call, so successive calls for the SAME eye of one ctx must be
 *                 ordered (same stream, or the caller's own events); the two eyes may run on different streams, and
 *                 frames in flight beyond that take one ctx each.
 * Lazy-initialises on first call and re-initialises when src dimensions change (:136-143).
 * Pass selection: upscale iff renderScale != 1; sharpen iff !useNis || renderScale == 1 (:586-594). */
OVRFSR_API int ovrfsr_apply(ovrfsr_ctx *ctx, int eye, const ovrfsr_image *src, int only_one_eye,
                            ovrfsr_image *out, void *stream);
/* Same pass with HOST images: copies src host->device, runs ovrfsr_apply, copies the result to
 * dst_host (which must be outW x outH of the ctx output format), all on `stream`.  Pinned host
 * memory makes the copies asynchronous.  This is the end-to-end entry bench.py times. */
OVRFSR_API int ovrfsr_apply_host(ovrfsr_ctx *ctx, int eye, const ovrfsr_image *src_host, int only_one_eye,
                                 const ovrfsr_image *dst_host, void *stream);

/* Both eyes of one frame in one call, for hosts that hold both textures when they submit (the reference's hook sees them
 * one Submit at a time, VrHooks.cpp:50-66; its D3D11 context is free to overlap the two eyes' dispatches, which have no
 * hazard between them -- a single CUDA stream is not).  Same result and same per-eye state as
 *   ovrfsr_apply(ctx, 0, src_left, only_one_eye, &out[0], stream); ovrfsr_apply(ctx, 1, src_right, only_one_eye, &out[1], stream);
 * but the right eye's passes run on a ctx-owned stream forked from `stream` before the left eye is queued and joined
 * back into it before the call returns, so the tail of one eye's launches overlaps the other eye's (C2, one caller
 * stream: see DESIGN.md section 7).  Everything queued on `stream` afterwards sees both outputs; capturable into a CUDA
 * graph.  With only_one_eye == 0 (one texture holding both eyes) it is exactly the two calls above. */
OVRFSR_API int ovrfsr_apply_pair(ovrfsr_ctx *ctx, const ovrfsr_image *src_left, const ovrfsr_image *src_right,
                                 int only_one_eye, ovrfsr_image out[2], void *stream);

/* ovrfsr_apply whose last pass writes the CALLER's image `dst` -- pitched device memory or a non-layered CUDA array
 * (OVRFSR_FORMAT_ARRAY_BIT), e.g. a texture the compositor can read -- instead of a ctx-owned output; the intermediates
 * stay ctx-owned.  dst must be outW x outH of the ctx output format (known after the lazy init, like ovrfsr_apply's
 * out; OVRFSR_ERR_INVALID otherwise).  With only_one_eye == 0 the shared texture is processed once, into the dst of the
 * call that processes it (the first Submit, PostProcessor.cpp:155-160): the second call writes nothing. */
OVRFSR_API int ovrfsr_apply_into(ovrfsr_ctx *ctx, int eye, const ovrfsr_image *src, int only_one_eye, const ovrfsr_image *dst,
                                 void *stream);
/* ovrfsr_apply_pair with ovrfsr_apply_into for each eye: dst[0] receives the left eye, dst[1] the right one. */
OVRFSR_API int ovrfsr_apply_pair_into(ovrfsr_ctx *ctx, const ovrfsr_image *src_left, const ovrfsr_image *src_right,
                                      int only_one_eye, const ovrfsr_image dst[2], void *stream);

/* ---- foveation: the radius mask follows the gaze ------------------------------------------
 * Focus of the radius mask for `eye`, in the same normalised coordinates as ovrfsr_config::proj_centre
 * (x right, y down, [0,1]; relative to the eye's half for a side-by-side texture).  Takes the place of that
 * eye's projection centre in the imageCentre words; the radius is unchanged.  No reset, no reallocation.
 * May be called from any thread, concurrently with the ctx's apply calls.  OVRFSR_ERR_INVALID for
 * eye not in {0,1} or x/y not finite or outside [0,1].
 * Late-latched: while some eye has a focus or a focus radius, or the sharpness is overridden (below), each apply
 * (every ovrfsr_apply* entry) starts with a 64-byte host->device copy of its eye's block on its stream -- the mask
 * words (imageCentre[4], the squared radius of each centre pair), RCAS's const0[0], the four sharpness words of the
 * NISConfig and padding -- and the kernels read them from device memory, so a frame uses the focus set before that
 * copy RUNS; a captured CUDA graph follows later calls on every replay.
 * Each (x, y) pair, the pair of radius words, the NIS strength pair (kSharpStrengthMin / Scale) and the NIS limit
 * pair (kSharpLimitMin / Scale) is published with one 64-bit store: a copy that overlaps an update may combine the
 * centre pairs of one update with the radius words of another, or the strength pair of one sharpness update with
 * the limit pair of another, each of them whole -- never the x of one update with the y of another -- and every
 * such combination is a valid set of words.  RCAS's sharpness is one word and cannot tear.
 * The focus survives ovrfsr_reset, ovrfsr_set_config and source-size changes.  Host memory only: no CUDA
 * call, no device needed. */
OVRFSR_API int ovrfsr_set_focus(ovrfsr_ctx *ctx, int eye, float x, float y);
/* Back to the projection centre for `eye` (the reference's behaviour); a focus radius stays.  Graphs captured
 * with a focus read the projection centre from then on; once no eye has a focus or a focus radius, applies stop
 * issuing the copy. */
OVRFSR_API int ovrfsr_clear_focus(ovrfsr_ctx *ctx, int eye);
/* Radius of eye's mask, in the units of ovrfsr_config::radius (R = uint(0.5 * radius * outH), host::centre_radius's
 * truncation).  Late-latched exactly like ovrfsr_set_focus; independent of it (a radius without a focus grows or
 * shrinks the circle around the projection centre).  For a side-by-side texture the left eye's radius applies to
 * the left centre and the right eye's to the right one.  Stored as given, so it survives ovrfsr_reset,
 * ovrfsr_set_config and source-size changes; a new ovrfsr_config::radius applies to eyes without one.  Lets a host
 * widen the mask while its gaze data cannot be trusted (blink, saccade, lost tracking) without a reset.
 * OVRFSR_ERR_INVALID for eye not in {0,1}, or radius not finite, negative or > 4 (R <= 2 * outH, so the kernels'
 * u32 square cannot wrap for outH <= 16384); the previous value stays.  Host memory only. */
OVRFSR_API int ovrfsr_set_focus_radius(ovrfsr_ctx *ctx, int eye, float radius);
/* back to ovrfsr_config::radius for eye; the focus stays */
OVRFSR_API int ovrfsr_clear_focus_radius(ovrfsr_ctx *ctx, int eye);
/* Sharpness of both eyes, in place of ovrfsr_config::sharpness, without a reset: what the sharpness hotkeys
 * (PostProcessor.cpp:670-704) or an in-headset slider change while the game runs.  Every apply entry point gives the
 * bytes of a ctx configured with that sharpness, in both math modes, on FSR (RCAS, alone or after EASU, fused or
 * not, with or without OVRFSR_FLAG_SRTM) and on NIS (NVScaler, NVSharpen).  Late-latched exactly like
 * ovrfsr_set_focus, in the same block.  Stored as given, so it survives ovrfsr_reset, ovrfsr_set_config and
 * source-size changes; a new ovrfsr_config::sharpness takes effect after ovrfsr_clear_sharpness.  An F7 capture
 * names its file with the override current when the capturing apply is issued.  ovrfsr_get_config,
 * ovrfsr_get_sharpen_constants and the stateless dispatches keep reporting / using the config's sharpness.
 * OVRFSR_ERR_INVALID for sharpness not finite or outside [0, 1]; the previous value stays.  Host memory only: any
 * thread, concurrently with applies, before the first one too. */
OVRFSR_API int ovrfsr_set_sharpness(ovrfsr_ctx *ctx, float sharpness);
/* back to ovrfsr_config::sharpness */
OVRFSR_API int ovrfsr_clear_sharpness(ovrfsr_ctx *ctx);

/* ---- individual dispatches (ApplyUpscaling / ApplySharpening, PostProcessor.cpp:385-401,483-496) --
 * Stateless: explicit constant blocks, caller-owned destination.  math_mode as ovrfsr_math. */
/* g_FSRUpscaleShader: consts = UpscaleConstants, 24 x u32 (PostProcessor.cpp:276-283) */
OVRFSR_API int ovrfsr_dispatch_fsr_easu(const ovrfsr_image *src, const ovrfsr_image *dst, const uint32_t consts[24],
                                        int math_mode, void *stream);
/* g_FSRSharpenShader: consts = SharpenConstants, 12 x u32 (PostProcessor.cpp:403-407) */
OVRFSR_API int ovrfsr_dispatch_fsr_rcas(const ovrfsr_image *src, const ovrfsr_image *dst, const uint32_t consts[12],
                                        int math_mode, void *stream);
/* The two dispatches above with the tone map of OVRFSR_FLAG_SRTM per pass (pass_flags, OR of the bits below), for hosts
 * that chain the passes themselves: F after the decode of every texel the pass reads, G before the encode of every pixel
 * it stores.  The ctx's chain is EASU with SRTM_IN into an RGBA16F / RGBA32F image, then RCAS with SRTM_OUT (RCAS alone:
 * both).  pass_flags == 0 launches exactly what ovrfsr_dispatch_fsr_easu / _rcas launch.  OVRFSR_ERR_UNSUPPORTED for
 * either bit with a UNORM source, OVRFSR_ERR_INVALID for unknown bits. */
#define OVRFSR_PASS_SRTM_IN 1
#define OVRFSR_PASS_SRTM_OUT 2
/* finite-in / finite-out of OVRFSR_FLAG_FINITE on the texels the pass reads / the pixels it stores, OR-ed with the SRTM
 * bits above (read: finite-in before F; store: G before finite-out) and accepted by all four _ex dispatches with the
 * same errors.  The ctx runs EASU with both, RCAS with both when its source is a float image, NVScaler / NVSharpen with
 * both, and the fused kernel (no stateless bits) with finite-in.  4 and 8 stay unknown bits (OVRFSR_ERR_INVALID), as
 * they were before these two existed. */
#define OVRFSR_PASS_FINITE_IN 16
#define OVRFSR_PASS_FINITE_OUT 32
/* perceptual-in / perceptual-out of OVRFSR_FLAG_PERCEPTUAL on the texels the pass reads / the pixels it stores, OR-ed
 * with the bits above (read: finite-in, F, then P; store: P^-1, G, then finite-out or the sRGB encode of an RGBA8 target)
 * and accepted by all four _ex dispatches with the same errors.  The ctx runs EASU with _IN, RCAS with _OUT after EASU
 * and with both alone, NVScaler / NVSharpen with both.  4, 8, 64 and 256 stay unknown bits (OVRFSR_ERR_INVALID). */
#define OVRFSR_PASS_PERCEPTUAL_IN 128
#define OVRFSR_PASS_PERCEPTUAL_OUT 512
OVRFSR_API int ovrfsr_dispatch_fsr_easu_ex(const ovrfsr_image *src, const ovrfsr_image *dst, const uint32_t consts[24],
                                           int math_mode, int pass_flags, void *stream);
OVRFSR_API int ovrfsr_dispatch_fsr_rcas_ex(const ovrfsr_image *src, const ovrfsr_image *dst, const uint32_t consts[12],
                                           int math_mode, int pass_flags, void *stream);
/* g_FSRUpscaleShader followed by g_FSRSharpenShader (ApplyPostProcess, PostProcessor.cpp:586-594) as ONE kernel: the
 * upscaled image is quantised to dst->format (RGBA8, or RGB10A2 for an RGB10A2 source) exactly as the first dispatch
 * stores it, but never leaves shared memory.  Bit-identical to the two dispatches above run back to back.  The two
 * constant blocks must carry the same centres / radius words (they do when built by ovrfsr_make_*_constants for one
 * eye); OVRFSR_ERR_UNSUPPORTED if this pair cannot be fused (formats, or a source
 * tile beyond the kernel's shared memory: out->in steps above about 0.85 in both axes, above about 1.03 in one). */
OVRFSR_API int ovrfsr_dispatch_fsr_fused(const ovrfsr_image *src, const ovrfsr_image *dst, const uint32_t upscale_consts[24],
                                         const uint32_t sharpen_consts[12], int math_mode, void *stream);
/* g_NISUpscaleShader / g_NISSharpenShader: cfg = NISConfig, 256 bytes (NIS_Config.h:37-77 + the
 * mod's centre/radius at byte 112, PostProcessor.cpp:310) */
OVRFSR_API int ovrfsr_dispatch_nis_scaler(const ovrfsr_image *src, const ovrfsr_image *dst, const void *cfg256,
                                          int math_mode, void *stream);
OVRFSR_API int ovrfsr_dispatch_nis_sharpen(const ovrfsr_image *src, const ovrfsr_image *dst, const void *cfg256,
                                           int math_mode, void *stream);
/* The two NIS dispatches above with the tone map of OVRFSR_FLAG_SRTM_NIS (pass_flags, OR of OVRFSR_PASS_SRTM_IN / _OUT,
 * and of OVRFSR_PASS_FINITE_IN / _OUT):
 * F after the decode of every texel the pass reads, G before the encode of every pixel it stores.  The ctx runs its one
 * NIS pass with both bits.  pass_flags == 0 launches exactly what ovrfsr_dispatch_nis_scaler / _sharpen launch.
 * OVRFSR_ERR_UNSUPPORTED for either bit with a UNORM source, OVRFSR_ERR_INVALID for unknown bits. */
OVRFSR_API int ovrfsr_dispatch_nis_scaler_ex(const ovrfsr_image *src, const ovrfsr_image *dst, const void *cfg256,
                                             int math_mode, int pass_flags, void *stream);
OVRFSR_API int ovrfsr_dispatch_nis_sharpen_ex(const ovrfsr_image *src, const ovrfsr_image *dst, const void *cfg256,
                                              int math_mode, int pass_flags, void *stream);

/* ---- host-side constant setup (pure CPU; usable without a GPU) -------------------------- */
/* PrepareResources, PostProcessor.cpp:509-518 */
OVRFSR_API void ovrfsr_output_size(uint32_t in_w, uint32_t in_h, float render_scale, uint32_t *out_w,
                                   uint32_t *out_h);
/* FsrEasuCon, ffx_fsr1.h:156-202 */
OVRFSR_API void ovrfsr_fsr_easu_con(uint32_t con[16], float in_vp_w, float in_vp_h, float in_w, float in_h,
                                    float out_w, float out_h);
/* FsrRcasCon, ffx_fsr1.h:662-672 (argument in stops) */
OVRFSR_API void ovrfsr_fsr_rcas_con(uint32_t con[4], float sharpness_stops);
/* UpscaleConstants for one eye, PostProcessor.cpp:293-305,331-337 */
OVRFSR_API void ovrfsr_make_upscale_constants(uint32_t consts[24], const ovrfsr_config *cfg, int eye,
                                              int only_one_eye, uint32_t in_w, uint32_t in_h, uint32_t out_w,
                                              uint32_t out_h);
/* SharpenConstants for one eye, PostProcessor.cpp:416-430,453-459 */
OVRFSR_API void ovrfsr_make_sharpen_constants(uint32_t consts[12], const ovrfsr_config *cfg, int eye,
                                              int only_one_eye, uint32_t out_w, uint32_t out_h);
/* NISConfig for one eye: NVScalerUpdateConfig (sharpen_only=0, PostProcessor.cpp:307-310) or
 * NVSharpenUpdateConfig (sharpen_only=1, :432-435).  Returns the bool the mod ignores (1 = scale in range). */
OVRFSR_API int ovrfsr_make_nis_config(void *cfg256, const ovrfsr_config *cfg, int sharpen_only, int eye,
                                      int only_one_eye, uint32_t in_w, uint32_t in_h, uint32_t out_w,
                                      uint32_t out_h);
/* coef_scale / coef_usm, NIS_Config.h:261-393: 64 phases x 8 floats */
OVRFSR_API const float *ovrfsr_nis_coef_scale(void);
OVRFSR_API const float *ovrfsr_nis_coef_usm(void);

/* ---- introspection -------------------------------------------------------------------- */
/* constant blocks the ctx built for `eye` (valid after the first apply) */
OVRFSR_API int ovrfsr_get_upscale_constants(const ovrfsr_ctx *ctx, int eye, uint32_t consts[24]);
OVRFSR_API int ovrfsr_get_sharpen_constants(const ovrfsr_ctx *ctx, int eye, uint32_t consts[12]);
/* Device self-test: strict-math RCAS replaces rcp.rn by MUFU.RCP + one Newton step when the source is UNORM8 (its
 * reciprocal operands then come from a set of 512 values); this runs both over the whole set on the current device.
 * *mismatches must come back 0. */
OVRFSR_API int ovrfsr_selftest_rcp(uint32_t *mismatches, uint32_t *checked);
/* Device self-test: strict-math NVScaler / NVSharpen with a UNORM source evaluate GetEdgeMap's and CalcLTI's quotients
 * (NIS_Scaler.h:244-247,373) with the in-range form of IEEE division (no exponent-range fallback); this compares it
 * with div.rn on ~19 M pseudo-random operand pairs of that range on the current device.  *mismatches must be 0. */
OVRFSR_API int ovrfsr_selftest_div(uint32_t *mismatches, uint32_t *checked);
/* kernels launched by this library in this process since load (bench.py's gpu_launches) */
OVRFSR_API uint64_t ovrfsr_kernel_launches(void);
/* debugMode profiling (PostProcessor.cpp:547-557,601-628): mean GPU ms per apply over the samples
 * collected so far (cudaEvent pairs read back a few frames late); returns samples used, 0 if none. */
OVRFSR_API int ovrfsr_get_gpu_time_ms(ovrfsr_ctx *ctx, float *mean_ms);
OVRFSR_API const char *ovrfsr_last_error(const ovrfsr_ctx *ctx);
OVRFSR_API const char *ovrfsr_status_string(int status);
OVRFSR_API uint32_t ovrfsr_version(void);
/* device image helpers (cudaMalloc with a 256-byte-aligned pitch, cudaFree) */
OVRFSR_API int ovrfsr_image_alloc(ovrfsr_image *img, uint32_t width, uint32_t height, int32_t format);
/* a CUDA-array image (cudaMalloc3DArray with the raw channel descriptor of `format`, cudaArraySurfaceLoadStore, and
 * cudaArrayLayered when layers > 1): img->format = format | OVRFSR_FORMAT_ARRAY_BIT */
OVRFSR_API int ovrfsr_image_alloc_array(ovrfsr_image *img, uint32_t width, uint32_t height, int32_t format, uint32_t layers);
/* frees either kind (an array after ovrfsr_release_array) */
OVRFSR_API void ovrfsr_image_free(ovrfsr_image *img);
/* dst <- src, two device images of the same size, format and slice count, each pitched or an array; all slices.
 * Asynchronous on `stream`.  OVRFSR_ERR_INVALID on a mismatch. */
OVRFSR_API int ovrfsr_image_copy(const ovrfsr_image *dst, const ovrfsr_image *src, void *stream);
/* Synchronises the device(s) the library used the array on and destroys the texture / surface objects it made for it.
 * Must be called before the array is freed: a freed handle that is reused for a new array would otherwise reach a
 * kernel through a stale object.  OVRFSR_ERR_INVALID if img is not an array image. */
OVRFSR_API int ovrfsr_release_array(const ovrfsr_image *img);


/* ---- the callers either side of the path (SURVEY.md 8f rows 2-4) -------------------------- */
/* R32G32B32_FLOAT source (PostProcessor.cpp:34-35) -> RGBA32F with alpha 1, what a shader reads from such a view.
 * src->format RGB32F (12-byte texels), dst->format RGBA32F, same size.  Asynchronous on `stream`. */
OVRFSR_API int ovrfsr_expand_rgb32f(const ovrfsr_image *src, const ovrfsr_image *dst, void *stream);
/* IsConsideredSrgbByOpenVR (PostProcessor.cpp:76-92) on a tagged ovrfsr_format: 1 for the _SRGB variants of RGBA8 /
 * BGRA8 / BGRX8 and for the _TYPELESS variants of RGBA8 / BGRA8 / BGRX8 / RGB10A2 */
OVRFSR_API int ovrfsr_format_considered_srgb(int32_t tagged_format);
/* GetInputView's MSAA branch (PostProcessor.cpp:219-226, ResolveSubresource): dst[x,y] = mean of the
 * sample_count samples of texel (x,y), same format in and out; src_samples laid out as ovrfsr_image::sample_count
 * describes (its width is the texel width).  Asynchronous on `stream`. */
OVRFSR_API int ovrfsr_resolve_msaa(const ovrfsr_image *src_samples, const ovrfsr_image *dst, void *stream);
/* IVRSystem_GetRecommendedRenderTargetSize detour (VrHooks.cpp:37-48): in/out the runtime's recommendation; scaled
 * by renderScale when fsr_enabled and renderScale < 1 (u32 *= float, truncating). */
OVRFSR_API void ovrfsr_recommended_render_size(const ovrfsr_config *cfg, uint32_t *width, uint32_t *height);
/* the MIP LOD bias handed to the sampler hook: -log2(outputWidth / (float)inputWidth), PostProcessor.cpp:537-538 */
OVRFSR_API float ovrfsr_mip_lod_bias(uint32_t input_width, uint32_t output_width);
/* D3D11Context_PSSetSamplers' rule (VrHooks.cpp:123-128): the bias a replacement sampler gets -- added only to
 * samplers without a bias of their own that filter anisotropically. */
OVRFSR_API float ovrfsr_sampler_lod_bias(float sampler_mip_lod_bias, uint32_t sampler_max_anisotropy, float mip_lod_bias);

/* The legacy CAS shaders the reference keeps under src/cas but never dispatches (src/CMakeLists.txt builds only fsr/
 * and nis/): CasSetup (src/cas/ffx_cas.h:375-397; consts = const0[4], const1[4]) and one CasFilter per output pixel,
 * alpha 1 (src/cas/cas.compute.h:25-47).  sharpen_only = cas.sharpen.hlsl (CAS_BETTER_DIAGONALS; dst size == src
 * size), else cas.upscale.hlsl (dst at least as large as src).  No radius mask exists on this path. */
OVRFSR_API void ovrfsr_cas_setup(uint32_t consts[8], float sharpness, float max_color_delta, float in_w, float in_h,
                                 float out_w, float out_h);
OVRFSR_API int ovrfsr_dispatch_cas(const ovrfsr_image *src, const ovrfsr_image *dst, const uint32_t consts[8],
                                   int sharpen_only, int math_mode, void *stream);

/* F7 capture (PostProcessor.cpp:630-657): the next apply for the LEFT eye writes its output image to
 * <directory>/capture_<YYYYmmdd_HHMMSS>_<fsr|nis>_s<sharpness*100>_r<radius*100>.dds and clears the request.
 * That apply synchronises the stream (the reference's SaveDDSTextureToFile maps a staging copy). */
OVRFSR_API int ovrfsr_request_capture(ovrfsr_ctx *ctx, const char *directory);
OVRFSR_API const char *ovrfsr_last_capture_path(const ovrfsr_ctx *ctx);
/* file name part of SaveTextureToFile (:641-652) for a given local time (seconds since the epoch) */
OVRFSR_API int ovrfsr_capture_filename(const ovrfsr_config *cfg, int64_t unix_time, char *buf, uint32_t buf_size);
/* DDS container exactly as ScreenGrab11's SaveDDSTextureToFile lays it out (ScreenGrab11.cpp:815-935): RGBA8 with
 * the legacy A8B8G8R8 masks, BGRA8 with A8R8G8B8, RGBA16F / RGBA32F as D3DFMT FourCC 113 / 116, RGB10A2 through the
 * 'DX10' extension header (dxgiFormat 24); one mip, tight rows.
 * host_image->data is HOST memory.  ovrfsr_dds_read allocates host_image->data (release with ovrfsr_host_free), so
 * a capture taken on a real D3D11 box can be diffed against this library's output. */
OVRFSR_API int ovrfsr_dds_write(const char *path, const ovrfsr_image *host_image);
OVRFSR_API int ovrfsr_dds_read(const char *path, ovrfsr_image *host_image);
OVRFSR_API void ovrfsr_host_free(void *p);

#ifdef __cplusplus
}
#endif
#endif /* OVRFSR_H */

/*
 * ovr_glue.h -- D3D11 fetch/store semantics and the entry-shader glue shared by
 * the restated oracle (oracle/ C files) and the compiled-reference driver
 * (oracle/ref_shim/ C++ files).  TEST INFRASTRUCTURE ONLY (see ovr_oracle.h).
 *
 * These are the parts of the path that live in D3D11 itself rather than in the
 * reference's source, restated once so that both checkers agree on them:
 *   Texture2D.Load        integer fetch, out-of-bounds -> 0     (fsr_rcas.hlsl:18)
 *   Gather{Red,Green,Blue} 2x2 footprint, clamp to edge, order
 *                          .w .z / .x .y                        (fsr_easu.hlsl:21-23,
 *                                                                ffx_fsr1.h:333-343)
 *   SampleLevel(linear clamp) bilinear, 8-bit sub-texel weights (fsr_easu.hlsl:34,
 *                                                                NIS_Upscale.hlsl:87)
 *   RWTexture2D store     float4 -> UNORM8 / FP16, bounds-checked (PostProcessor.cpp:340-358)
 */
#ifndef OVR_GLUE_H
#define OVR_GLUE_H

#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "ovr_oracle.h"

static inline float ovo_u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t ovo_f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

/* HLSL min / max / saturate.  D3D11 pins NaN handling (the other operand; saturate(NaN) = 0) and leaves the sign of
 * min(+0, -0) to the implementation; C's fminf / fmaxf leave it open too (glibc returns the first operand).  The checker
 * pins the rule sm_90a's FMNMX follows, which tests/test_gpu_minmax_rule.py measures on the device: IEEE 754-2019
 * minimumNumber / maximumNumber -- NaN ignored, -0 < +0, independent of operand order.  No libm call: the bits must
 * not depend on the host's C library.  saturate(x) = min(1, max(+0, x)), so saturate(-0) = +0 (FADD.SAT: +0 + -0). */
static inline float ovo_min(float a, float b) {
  if (a != a) return b;
  if (b != b) return a;
  if (a != b) return a < b ? a : b;
  return (ovo_f2u(a) & 0x80000000u) ? a : b; /* equal: only a zero pair can differ in bits; -0 wins */
}
static inline float ovo_max(float a, float b) {
  if (a != a) return b;
  if (b != b) return a;
  if (a != b) return a > b ? a : b;
  return (ovo_f2u(a) & 0x80000000u) ? b : a; /* equal: +0 wins */
}
static inline float ovo_sat(float a) { return ovo_min(1.0f, ovo_max(0.0f, a)); }

/* IEEE half <-> float (exact up-conversion, round-to-nearest-even down-conversion) */
static inline float ovo_half_to_float(uint16_t h) {
  uint32_t s = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 0x1fu, m = h & 0x3ffu;
  if (e == 0) {
    if (m == 0) return ovo_u2f(s);
    float f = (float)m * (1.0f / 16777216.0f); /* m * 2^-24, exact */
    return s ? -f : f;
  }
  if (e == 31) return ovo_u2f(s | 0x7f800000u | (m << 13));
  return ovo_u2f(s | ((e + 112u) << 23) | (m << 13));
}
static inline uint16_t ovo_float_to_half(float f) {
  uint32_t u = ovo_f2u(f), s = (u >> 16) & 0x8000u;
  u &= 0x7fffffffu;
  if (u > 0x7f800000u) return (uint16_t)(s | 0x7e00u);            /* NaN */
  if (u >= 0x477ff000u) return (uint16_t)(s | 0x7c00u);           /* >= 65520 -> inf */
  if (u < 0x33000001u) return (uint16_t)s;                        /* <= 2^-25 -> 0 */
  if (u < 0x38800000u) {                                          /* subnormal half */
    uint32_t sh = 126u - (u >> 23), m = (u & 0x7fffffu) | 0x800000u;
    uint32_t r = m >> sh, rem = m & ((1u << sh) - 1u), half = 1u << (sh - 1u);
    if (rem > half || (rem == half && (r & 1u))) r++;
    return (uint16_t)(s | r);
  }
  uint32_t r = u - 0x38000000u, rem = r & 0x1fffu;
  r >>= 13;
  if (rem > 0x1000u || (rem == 0x1000u && (r & 1u))) r++;
  return (uint16_t)(s | r);
}

/* ffx_a.h:482-550 AU1_AH1_AF1: table-driven float->half that TRUNCATES the
 * mantissa and clamps overflow/inf/NaN to 0x7bff.  The 2x512-entry tables are
 * regenerated here from their construction rule instead of being listed. */
static inline uint32_t ovo_half_bits_trunc(float f) {
  uint32_t u = ovo_f2u(f), i = u >> 23, e = i & 0xffu, sign = (i & 0x100u) ? 0x8000u : 0u;
  uint32_t base, shift;
  if (e < 103u) { base = 0; shift = 24; }
  else if (e < 113u) { base = 0x0400u >> (113u - e); shift = 126u - e; }
  else if (e <= 142u) { base = (e - 112u) << 10; shift = 13; }
  else { base = 0x7bffu; shift = 24; }
  return (base | sign) + ((u & 0x7fffffu) >> shift);
}

static inline int ovo_bpp(int format) {
  return format == OVO_FMT_RGBA32F ? 16 : (format == OVO_FMT_RGB32F ? 12 : (format == OVO_FMT_RGBA16F ? 8 : 4));
}

/* in-bounds texel fetch -> float4 (rgba) */
static inline void ovo_texel(const ovo_image *im, int x, int y, float o[4]) {
  const uint8_t *row = (const uint8_t *)im->data + (size_t)y * (size_t)im->pitch;
  if (im->format == OVO_FMT_RGBA32F) {
    memcpy(o, row + (size_t)x * 16, 16);
  } else if (im->format == OVO_FMT_RGB32F) { /* a missing component reads as 1 in alpha (D3D11 default for .w) */
    memcpy(o, row + (size_t)x * 12, 12);
    o[3] = 1.0f;
  } else if (im->format == OVO_FMT_RGBA16F) {
    const uint16_t *p = (const uint16_t *)(row + (size_t)x * 8);
    o[0] = ovo_half_to_float(p[0]); o[1] = ovo_half_to_float(p[1]);
    o[2] = ovo_half_to_float(p[2]); o[3] = ovo_half_to_float(p[3]);
  } else if (im->format == OVO_FMT_RGB10A2) {
    uint32_t p;
    memcpy(&p, row + (size_t)x * 4, 4);
    o[0] = (float)(p & 1023u) / 1023.0f; o[1] = (float)((p >> 10) & 1023u) / 1023.0f;
    o[2] = (float)((p >> 20) & 1023u) / 1023.0f; o[3] = (float)(p >> 30) / 3.0f;
  } else {
    const uint8_t *p = row + (size_t)x * 4;
    float a = (float)p[0] / 255.0f, b = (float)p[1] / 255.0f, c = (float)p[2] / 255.0f;
    o[3] = im->format == OVO_FMT_BGRX8 ? 1.0f : (float)p[3] / 255.0f; /* X8: alpha reads as 1 */
    o[1] = b;
    if (im->format == OVO_FMT_BGRA8 || im->format == OVO_FMT_BGRX8) { o[0] = c; o[2] = a; } else { o[0] = a; o[2] = c; }
  }
}

/* Texture2D.Load / operator[]: out-of-bounds returns 0 */
static inline void ovo_load(const ovo_image *im, int x, int y, float o[4]) {
  if (x < 0 || y < 0 || x >= im->width || y >= im->height) { o[0] = o[1] = o[2] = o[3] = 0.0f; return; }
  ovo_texel(im, x, y, o);
}

/* clamp-to-edge fetch (sampler address mode CLAMP) */
static inline void ovo_texel_clamp(const ovo_image *im, int x, int y, float o[4]) {
  x = x < 0 ? 0 : (x >= im->width ? im->width - 1 : x);
  y = y < 0 ? 0 : (y >= im->height ? im->height - 1 : y);
  ovo_texel(im, x, y, o);
}

/* SampleLevel(linearClamp, uv, 0): bilinear at normalised uv.  D3D11 converts the scaled texture
 * coordinate to fixed point with 8 fractional bits before filtering (functional spec 7.18.8 /
 * D3D11_SUBTEXEL_FRACTIONAL_BIT_COUNT = 8), which every D3D11 GPU implements: the coordinate is snapped
 * to 1/256 texel (round to nearest), so weights are multiples of 1/256 and a sample aimed at a texel
 * centre returns exactly that texel (NVScaler relies on this for its luma taps, NIS_Scaler.h:642-651). */
static inline float ovo_snap_subtexel(float s) { return floorf(s * 256.0f + 0.5f) * (1.0f / 256.0f); }
static inline void ovo_sample_linear(const ovo_image *im, float u, float v, float o[4]) {
  float sx = ovo_snap_subtexel(u * (float)im->width - 0.5f), sy = ovo_snap_subtexel(v * (float)im->height - 0.5f);
  float fx0 = floorf(sx), fy0 = floorf(sy);
  float fx = sx - fx0, fy = sy - fy0;
  int x0 = (int)fx0, y0 = (int)fy0;
  float c00[4], c10[4], c01[4], c11[4];
  ovo_texel_clamp(im, x0, y0, c00);
  ovo_texel_clamp(im, x0 + 1, y0, c10);
  ovo_texel_clamp(im, x0, y0 + 1, c01);
  ovo_texel_clamp(im, x0 + 1, y0 + 1, c11);
  float wx0 = 1.0f - fx, wy0 = 1.0f - fy;
  for (int i = 0; i < 4; ++i) {
    float top = c00[i] * wx0 + c10[i] * fx;
    float bot = c01[i] * wx0 + c11[i] * fx;
    o[i] = top * wy0 + bot * fy;
  }
}

/* RWTexture2D store with UAV bounds check */
static inline void ovo_store(const ovo_image *im, int x, int y, const float c[4]) {
  if (x < 0 || y < 0 || x >= im->width || y >= im->height) return;
  uint8_t *row = (uint8_t *)im->data + (size_t)y * (size_t)im->pitch;
  if (im->format == OVO_FMT_RGBA32F) {
    memcpy(row + (size_t)x * 16, c, 16);
  } else if (im->format == OVO_FMT_RGBA16F) {
    uint16_t *p = (uint16_t *)(row + (size_t)x * 8);
    for (int i = 0; i < 4; ++i) p[i] = ovo_float_to_half(c[i]);
  } else if (im->format == OVO_FMT_RGB10A2) {
    uint32_t p = (uint32_t)(ovo_sat(c[0]) * 1023.0f + 0.5f) | ((uint32_t)(ovo_sat(c[1]) * 1023.0f + 0.5f) << 10) |
                 ((uint32_t)(ovo_sat(c[2]) * 1023.0f + 0.5f) << 20) | ((uint32_t)(ovo_sat(c[3]) * 3.0f + 0.5f) << 30);
    memcpy(row + (size_t)x * 4, &p, 4);
  } else {
    uint8_t *p = row + (size_t)x * 4;
    uint8_t q[4];
    for (int i = 0; i < 4; ++i) q[i] = (uint8_t)(ovo_sat(c[i]) * 255.0f + 0.5f);
    if (im->format == OVO_FMT_BGRA8) { p[0] = q[2]; p[1] = q[1]; p[2] = q[0]; p[3] = q[3]; }
    else { p[0] = q[0]; p[1] = q[1]; p[2] = q[2]; p[3] = q[3]; }
  }
}

/* workgroup radius test, fsr_easu.hlsl:40-44 / NIS_Upscale.hlsl:98-101: wrapping u32 arithmetic */
static inline int ovo_group_inside_(uint32_t gx, uint32_t gy, uint32_t gw, uint32_t gh, const uint32_t centre[4],
                                    uint32_t radiusSq) {
  uint32_t cx = gx * gw + (gw >> 1), cy = gy * gh + (gh >> 1);
  uint32_t d1x = centre[0] - cx, d1y = centre[1] - cy;
  uint32_t d2x = centre[2] - cx, d2y = centre[3] - cy;
  uint32_t dd1 = d1x * d1x + d1y * d1y, dd2 = d2x * d2x + d2y * d2y;
  return dd1 <= radiusSq || dd2 <= radiusSq;
}

/* ---- row-parallel runner (work-stealing over row chunks) ---------------- */
typedef void (*ovo_rows_fn)(void *arg, int y0, int y1);
typedef struct { ovo_rows_fn fn; void *arg; int rows, chunk; volatile int next; } ovo_par_;
static void *ovo_par_worker_(void *p) {
  ovo_par_ *s = (ovo_par_ *)p;
  for (;;) {
    int y0 = __sync_fetch_and_add(&s->next, s->chunk);
    if (y0 >= s->rows) break;
    int y1 = y0 + s->chunk; if (y1 > s->rows) y1 = s->rows;
    s->fn(s->arg, y0, y1);
  }
  return 0;
}
static inline int ovo_parallel_rows(int rows, int chunk, int nthreads, ovo_rows_fn fn, void *arg) {
  ovo_par_ s; s.fn = fn; s.arg = arg; s.rows = rows; s.chunk = chunk; s.next = 0;
  if (nthreads <= 1) { ovo_par_worker_(&s); return 0; }
  if (nthreads > 512) nthreads = 512;
  pthread_t *t = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nthreads);
  if (!t) return -1;
  int n = 0;
  for (; n < nthreads - 1; ++n) if (pthread_create(&t[n], 0, ovo_par_worker_, &s)) break;
  ovo_par_worker_(&s);
  for (int i = 0; i < n; ++i) pthread_join(t[i], 0);
  free(t);
  return 0;
}

#endif

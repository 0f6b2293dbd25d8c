/*
 * selfcheck.c -- runs every pass of the restated oracle on small, ragged images; meant to be built with
 * -fsanitize=address,undefined (make -C oracle selfcheck) so that an out-of-bounds read or undefined operation in
 * the CHECKER itself cannot hide behind a lucky comparison.  TEST INFRASTRUCTURE ONLY (tests/test_oracle_sanitized.py).
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "ovr_oracle.h"

static uint32_t rng_state = 12345u;
static uint32_t rnd(void) { rng_state = rng_state * 1664525u + 1013904223u; return rng_state >> 8; }

/* the non-finite words a float eye texture can hold: +-inf, quiet and signalling NaNs with payloads, of both signs */
static const uint16_t kHalfNonFinite[] = {0x7c00u, 0xfc00u, 0x7e00u, 0xfe00u, 0x7c01u, 0xfdffu};
static const uint32_t kFloatNonFinite[] = {0x7f800000u, 0xff800000u, 0x7fc00000u, 0xffc00000u, 0x7f800001u,
                                           0xff800001u, 0x7fc00001u};

/* fill: 0 none, 1 random bytes (finite halves), 2 random finite content with about one word in 16 non-finite */
static ovo_image make(int w, int h, int fmt, int fill) {
  ovo_image im;
  const int bpp = fmt == OVO_FMT_RGBA32F ? 16 : (fmt == OVO_FMT_RGBA16F ? 8 : 4);
  im.width = w; im.height = h; im.pitch = w * bpp; im.format = fmt;
  im.data = malloc((size_t)im.pitch * (size_t)h); /* exact size: any overrun is caught by ASan */
  if (fill) {
    uint8_t *p = (uint8_t *)im.data;
    for (size_t i = 0; i < (size_t)im.pitch * (size_t)h; ++i) p[i] = (uint8_t)rnd();
    if (fmt == OVO_FMT_RGBA16F && fill == 1) { /* keep the halves finite and below 2: clear the top exponent bit */
      uint16_t *q = (uint16_t *)im.data;
      for (size_t i = 0; i < (size_t)w * (size_t)h * 4; ++i) q[i] &= 0xbbffu;
    }
    if (fill == 2 && fmt == OVO_FMT_RGBA16F) {
      uint16_t *q = (uint16_t *)im.data;
      for (size_t i = 0; i < (size_t)w * (size_t)h * 4; ++i) /* random finite halves up to 65504, and non-finite words */
        q[i] = (rnd() & 15u) == 0 ? kHalfNonFinite[rnd() % 6u] : (uint16_t)(((q[i] & 0x7c00u) == 0x7c00u ? q[i] & 0xbfffu : q[i]));
    } else if (fill == 2 && fmt == OVO_FMT_RGBA32F) {
      uint32_t *q = (uint32_t *)im.data;
      for (size_t i = 0; i < (size_t)w * (size_t)h * 4; ++i) {
        const uint32_t r = rnd();
        /* otherwise the random word, any finite float (subnormals and values up to 3.4e38 beyond the encodes' range);
           an exponent of all ones loses its top bit */
        q[i] = (r & 15u) == 0 ? kFloatNonFinite[(r >> 4) % 7u]
                              : ((q[i] & 0x7f800000u) == 0x7f800000u ? q[i] & 0xbfffffffu : q[i]);
      }
    }
  }
  return im;
}

int main(void) {
  static const int sizes[][2] = {{1, 1}, {2, 3}, {5, 4}, {16, 16}, {17, 13}, {33, 47}, {64, 24}};
  static const float scales[] = {0.5f, 0.59f, 0.75f, 1.0f, 1.3f};
  /* the float formats twice: random finite content, then the same with non-finite words (OVO_NONFINITE) */
  enum { OVO_NONFINITE = 0x100 };
  static const int fmts[] = {OVO_FMT_RGBA8, OVO_FMT_BGRA8, OVO_FMT_RGBA16F, OVO_FMT_RGB10A2,
                             OVO_FMT_RGBA16F | OVO_NONFINITE, OVO_FMT_RGBA32F | OVO_NONFINITE};
  const float proj[4] = {0.45f, 0.52f, 0.55f, 0.48f};
  int runs = 0;
  for (unsigned si = 0; si < sizeof(sizes) / sizeof(sizes[0]); ++si)
    for (unsigned ci = 0; ci < sizeof(scales) / sizeof(scales[0]); ++ci)
      for (unsigned fi = 0; fi < sizeof(fmts) / sizeof(fmts[0]); ++fi) {
        const int iw = sizes[si][0], ih = sizes[si][1], fmt = fmts[fi] & 0xff, fill = fmts[fi] & OVO_NONFINITE ? 2 : 1;
        const float scale = scales[ci], radius = (runs & 1) ? 0.4f : 2.0f;
        uint32_t ow, oh;
        ovo_output_size((uint32_t)iw, (uint32_t)ih, scale, &ow, &oh);
        if (ow == 0 || oh == 0) continue;
        /* non-finite content goes to every target format: UNORM8 / 10-bit (the encode's saturate), FP16, FP32 */
        static const int kOut[] = {OVO_FMT_RGBA8, OVO_FMT_RGBA16F, OVO_FMT_RGBA32F, OVO_FMT_RGB10A2};
        const int ofmt = fill == 2 ? kOut[runs & 3]
                                   : (fmt == OVO_FMT_RGB10A2 ? OVO_FMT_RGB10A2 : ((runs & 2) ? OVO_FMT_RGBA32F : OVO_FMT_RGBA8));
        ovo_image src = make(iw, ih, fmt, fill), mid = make((int)ow, (int)oh, ofmt, 0), dst = make((int)ow, (int)oh, ofmt, 0);
        ovo_upscale_constants uc;
        ovo_sharpen_constants sc;
        ovo_make_upscale_constants(&uc, runs & 1, 1, (uint32_t)iw, (uint32_t)ih, ow, oh, proj, radius);
        ovo_make_sharpen_constants(&sc, runs & 1, 1, ow, oh, proj, radius, 0.9f, runs & 4);
        if (ovo_fsr_easu(&src, &mid, &uc, 2) != 0 || ovo_fsr_rcas(&mid, &dst, &sc, 2) != 0) { puts("FSR pass failed"); return 1; }
        if (fill == 2) { /* RCAS on the source itself: the float -> target encode that tests/srtm_oracle.py composes with */
          ovo_image same = make(iw, ih, ofmt, 0);
          ovo_sharpen_constants ss;
          ovo_make_sharpen_constants(&ss, runs & 1, 1, (uint32_t)iw, (uint32_t)ih, proj, radius, 0.9f, runs & 4);
          if (ovo_fsr_rcas(&src, &same, &ss, 1) != 0) { puts("RCAS pass failed"); return 1; }
          free(same.data);
        }
        if (scale <= 1.0f && fmt != OVO_FMT_RGB10A2) {
          ovo_nis_config nc;
          ovo_cas_constants cc;
          ovo_make_nis_config(&nc, scale == 1.0f, runs & 1, 1, (uint32_t)iw, (uint32_t)ih, ow, oh, proj, radius, 0.7f, runs & 4);
          if ((scale == 1.0f ? ovo_nis_sharpen(&src, &dst, &nc, 2) : ovo_nis_scaler(&src, &dst, &nc, 2)) != 0) { puts("NIS pass failed"); return 1; }
          ovo_cas_setup(&cc, 0.8f, (runs & 8) ? 0.1f : 1.0f, (float)iw, (float)ih, (float)ow, (float)oh);
          if (ovo_cas(&src, &dst, &cc, scale == 1.0f, 2) != 0) { puts("CAS pass failed"); return 1; }
          if (ovo_cas(&src, &dst, &cc, 0, 1) != 0) { puts("CAS upscale pass failed"); return 1; }
        }
        free(src.data); free(mid.data); free(dst.data);
        ++runs;
      }
  printf("oracle selfcheck: %d configurations ok\n", runs);
  return 0;
}

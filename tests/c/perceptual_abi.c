/* perceptual_abi.c -- OVRFSR_FLAG_PERCEPTUAL and the OVRFSR_PASS_PERCEPTUAL_* bits of the four _ex dispatches from plain
 * C (C11, -pedantic), host work only: the flag round-trips through a ctx's config, and the dispatches refuse their
 * arguments before any launch (the image addresses below are never dereferenced).  Built and run by
 * tests/test_perceptual_host.py.  Prints one line per failed check; exit code 0 = all good. */
#include <stdio.h>
#include <string.h>

#include "ovrfsr.h"

static int fails = 0;
#define CHECK(cond) do { if (!(cond)) { printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #cond); ++fails; } } while (0)

static ovrfsr_image fake(int fmt, uint32_t w, uint32_t h, uintptr_t addr) {
  ovrfsr_image im;
  const uint32_t bpp = fmt == OVRFSR_FORMAT_RGBA32F ? 16u : (fmt == OVRFSR_FORMAT_RGBA16F ? 8u : 4u);
  memset(&im, 0, sizeof(im));
  im.data = (void *)addr; im.width = w; im.height = h; im.pitch = w * bpp; im.format = fmt; im.array_slices = 1;
  return im;
}

int main(void) {
  ovrfsr_config cfg, got;
  ovrfsr_ctx *ctx = NULL;
  unsigned char nis[256];
  uint32_t ku[24], ks[12];
  const int perc = OVRFSR_PASS_PERCEPTUAL_IN | OVRFSR_PASS_PERCEPTUAL_OUT;
  const int all = OVRFSR_PASS_SRTM_IN | OVRFSR_PASS_SRTM_OUT | OVRFSR_PASS_FINITE_IN | OVRFSR_PASS_FINITE_OUT | perc;
  ovrfsr_image s16 = fake(OVRFSR_FORMAT_RGBA16F, 64, 32, 0x7f0000000000u), d16 = fake(OVRFSR_FORMAT_RGBA16F, 64, 32, 0x7f0000100000u);
  ovrfsr_image s8 = fake(OVRFSR_FORMAT_RGBA8, 64, 32, 0x7f0000000000u), d8 = fake(OVRFSR_FORMAT_RGBA8, 64, 32, 0x7f0000100000u);
  int flags;

  CHECK(OVRFSR_FLAG_PERCEPTUAL == 16 &&
        (OVRFSR_FLAG_PERCEPTUAL & (OVRFSR_FLAG_FUSED_FSR | OVRFSR_FLAG_SRTM | OVRFSR_FLAG_SRTM_NIS | OVRFSR_FLAG_FINITE)) == 0);
  CHECK(OVRFSR_PASS_PERCEPTUAL_IN == 128 && OVRFSR_PASS_PERCEPTUAL_OUT == 512);
  CHECK((perc & (OVRFSR_PASS_SRTM_IN | OVRFSR_PASS_SRTM_OUT | OVRFSR_PASS_FINITE_IN | OVRFSR_PASS_FINITE_OUT)) == 0);
  ovrfsr_config_default(&cfg);
  cfg.fsr_enabled = 1; cfg.render_scale = 0.75f;
  cfg.flags = OVRFSR_FLAG_PERCEPTUAL;
  CHECK(ovrfsr_create(&ctx, &cfg) == OVRFSR_OK && ctx != NULL);
  CHECK(ovrfsr_get_config(ctx, &got) == OVRFSR_OK && got.flags == OVRFSR_FLAG_PERCEPTUAL);
  cfg.flags = OVRFSR_FLAG_PERCEPTUAL | OVRFSR_FLAG_SRTM | OVRFSR_FLAG_FINITE;
  CHECK(ovrfsr_set_config(ctx, &cfg) == OVRFSR_OK);
  CHECK(ovrfsr_get_config(ctx, &got) == OVRFSR_OK && got.flags == (OVRFSR_FLAG_PERCEPTUAL | OVRFSR_FLAG_SRTM | OVRFSR_FLAG_FINITE));
  ovrfsr_destroy(ctx);
  /* a tagged sRGB RGBA8 image reads as sRGB */
  CHECK(ovrfsr_format_considered_srgb(OVRFSR_FORMAT_RGBA8 | OVRFSR_FORMAT_SRGB_BIT) == 1);

  memset(nis, 0, sizeof(nis));
  memset(ku, 0, sizeof(ku));
  memset(ks, 0, sizeof(ks));
  CHECK(ovrfsr_make_nis_config(nis, &cfg, 1, 0, 1, 64, 32, 64, 32) == 1);
  /* either perceptual bit, alone or with the other known bits, on a UNORM source */
  for (flags = 1; flags <= all; ++flags) {
    if ((flags & ~all) || !(flags & perc)) continue;
    CHECK(ovrfsr_dispatch_fsr_easu_ex(&s8, &d8, ku, OVRFSR_MATH_STRICT, flags, NULL) == OVRFSR_ERR_UNSUPPORTED);
    CHECK(ovrfsr_dispatch_fsr_rcas_ex(&s8, &d8, ks, OVRFSR_MATH_FAST, flags, NULL) == OVRFSR_ERR_UNSUPPORTED);
    CHECK(ovrfsr_dispatch_nis_scaler_ex(&s8, &d8, nis, OVRFSR_MATH_STRICT, flags, NULL) == OVRFSR_ERR_UNSUPPORTED);
    CHECK(ovrfsr_dispatch_nis_sharpen_ex(&s8, &d8, nis, OVRFSR_MATH_FAST, flags, NULL) == OVRFSR_ERR_UNSUPPORTED);
  }
  /* bits beside the six known ones (4, 8, 64, 256, 1024, ...), with the perceptual bits on a float source */
  for (flags = 4; flags <= 4096; flags *= 2) {
    if (flags & all) continue;
    CHECK(ovrfsr_dispatch_fsr_easu_ex(&s16, &d16, ku, OVRFSR_MATH_STRICT, flags | perc, NULL) == OVRFSR_ERR_INVALID);
    CHECK(ovrfsr_dispatch_fsr_rcas_ex(&s16, &d16, ks, OVRFSR_MATH_STRICT, flags | perc, NULL) == OVRFSR_ERR_INVALID);
    CHECK(ovrfsr_dispatch_nis_scaler_ex(&s16, &d16, nis, OVRFSR_MATH_STRICT, flags | perc, NULL) == OVRFSR_ERR_INVALID);
    CHECK(ovrfsr_dispatch_nis_sharpen_ex(&s16, &d16, nis, OVRFSR_MATH_FAST, flags | perc, NULL) == OVRFSR_ERR_INVALID);
  }
  printf(fails ? "perceptual_abi: %d check(s) failed\n" : "perceptual_abi: ok\n", fails);
  return fails ? 1 : 0;
}

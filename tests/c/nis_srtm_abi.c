/* nis_srtm_abi.c -- OVRFSR_FLAG_SRTM_NIS and ovrfsr_dispatch_nis_scaler_ex / _sharpen_ex from plain C (C11, -pedantic),
 * host work only: the flag round-trips through a ctx's config, and the dispatches refuse their arguments before any
 * launch (the image addresses below are never dereferenced).  Built and run by tests/test_nis_srtm_host.py.
 * Prints one line per failed check; exit code 0 = all good. */
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
  ovrfsr_image s16 = fake(OVRFSR_FORMAT_RGBA16F, 64, 32, 0x7f0000000000u), d16 = fake(OVRFSR_FORMAT_RGBA16F, 64, 32, 0x7f0000100000u);
  ovrfsr_image s8 = fake(OVRFSR_FORMAT_RGBA8, 64, 32, 0x7f0000000000u), d8 = fake(OVRFSR_FORMAT_RGBA8, 64, 32, 0x7f0000100000u);
  int flags;

  CHECK(OVRFSR_FLAG_SRTM_NIS == 4 && (OVRFSR_FLAG_SRTM_NIS & (OVRFSR_FLAG_SRTM | OVRFSR_FLAG_FUSED_FSR)) == 0);
  ovrfsr_config_default(&cfg);
  cfg.fsr_enabled = 1; cfg.use_nis = 1; cfg.render_scale = 0.75f;
  cfg.flags = OVRFSR_FLAG_SRTM_NIS;
  CHECK(ovrfsr_create(&ctx, &cfg) == OVRFSR_OK && ctx != NULL);
  CHECK(ovrfsr_get_config(ctx, &got) == OVRFSR_OK && got.flags == OVRFSR_FLAG_SRTM_NIS);
  cfg.flags = OVRFSR_FLAG_SRTM_NIS | OVRFSR_FLAG_SRTM;
  CHECK(ovrfsr_set_config(ctx, &cfg) == OVRFSR_OK);
  CHECK(ovrfsr_get_config(ctx, &got) == OVRFSR_OK && got.flags == (OVRFSR_FLAG_SRTM_NIS | OVRFSR_FLAG_SRTM));
  ovrfsr_destroy(ctx);

  memset(nis, 0, sizeof(nis));
  CHECK(ovrfsr_make_nis_config(nis, &cfg, 1, 0, 1, 64, 32, 64, 32) == 1);
  for (flags = OVRFSR_PASS_SRTM_IN; flags <= (OVRFSR_PASS_SRTM_IN | OVRFSR_PASS_SRTM_OUT); ++flags) {
    CHECK(ovrfsr_dispatch_nis_scaler_ex(&s8, &d8, nis, OVRFSR_MATH_STRICT, flags, NULL) == OVRFSR_ERR_UNSUPPORTED);
    CHECK(ovrfsr_dispatch_nis_sharpen_ex(&s8, &d8, nis, OVRFSR_MATH_FAST, flags, NULL) == OVRFSR_ERR_UNSUPPORTED);
  }
  CHECK(ovrfsr_dispatch_nis_scaler_ex(&s16, &d16, nis, OVRFSR_MATH_STRICT, 4, NULL) == OVRFSR_ERR_INVALID);
  CHECK(ovrfsr_dispatch_nis_sharpen_ex(&s16, &d16, nis, OVRFSR_MATH_STRICT, -1, NULL) == OVRFSR_ERR_INVALID);
  CHECK(ovrfsr_dispatch_nis_scaler_ex(&s16, &d16, NULL, OVRFSR_MATH_STRICT, OVRFSR_PASS_SRTM_IN, NULL) == OVRFSR_ERR_INVALID);
  printf(fails ? "nis_srtm_abi: %d check(s) failed\n" : "nis_srtm_abi: ok\n", fails);
  return fails ? 1 : 0;
}

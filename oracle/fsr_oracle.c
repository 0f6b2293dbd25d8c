/*
 * fsr_oracle.c -- CPU restatement of the FSR1 half of the openvr_fsr hot path:
 * constant setup, EASU (edge-adaptive spatial upsampling) and RCAS (robust
 * contrast-adaptive sharpening), one scalar function per reference function,
 * same operation order so that results are bit-identical to the reference's
 * own lines compiled on the host (oracle/_ref, see build_ref.sh).
 *
 * TEST INFRASTRUCTURE ONLY -- see ovr_oracle.h for who may use this file.
 * Build: gcc -O2 -ffp-contract=off (no FMA fusion).  Citations: /root/reference/.
 */
#include "ovr_glue.h"

/* ------------------------------------------------------------------------
 * constants
 * ---------------------------------------------------------------------- */

/* PostProcessor.cpp:512-518: uint / float -> float -> uint (truncation) */
void ovo_output_size(uint32_t inW, uint32_t inH, float renderScale, uint32_t *outW, uint32_t *outH) {
  if (renderScale < 1.f) {
    *outW = (uint32_t)((float)inW / renderScale);
    *outH = (uint32_t)((float)inH / renderScale);
  } else {
    *outW = (uint32_t)((float)inW * renderScale);
    *outH = (uint32_t)((float)inH * renderScale);
  }
}

/* ffx_a.h:326 ARcpF1 on the CPU is a true divide */
static inline float rcpf(float a) { return 1.0f / a; }

/* ffx_fsr1.h:156-202.  Every product is "x * rcp(y)", never "x / y". */
void ovo_fsr_easu_con(uint32_t con[16], float inVpW, float inVpH, float inW, float inH, float outW, float outH) {
  con[0] = ovo_f2u(inVpW * rcpf(outW));
  con[1] = ovo_f2u(inVpH * rcpf(outH));
  con[2] = ovo_f2u(0.5f * inVpW * rcpf(outW) - 0.5f);
  con[3] = ovo_f2u(0.5f * inVpH * rcpf(outH) - 0.5f);
  con[4] = ovo_f2u(rcpf(inW));
  con[5] = ovo_f2u(rcpf(inH));
  con[6] = ovo_f2u(1.0f * rcpf(inW));
  con[7] = ovo_f2u(-1.0f * rcpf(inH));
  con[8] = ovo_f2u(-1.0f * rcpf(inW));
  con[9] = ovo_f2u(2.0f * rcpf(inH));
  con[10] = ovo_f2u(1.0f * rcpf(inW));
  con[11] = ovo_f2u(2.0f * rcpf(inH));
  con[12] = ovo_f2u(0.0f * rcpf(inW));
  con[13] = ovo_f2u(4.0f * rcpf(inH));
  con[14] = con[15] = 0;
}

/* ffx_fsr1.h:662-672 */
void ovo_fsr_rcas_con(uint32_t con[4], float sharpnessStops) {
  float s = exp2f(-sharpnessStops);
  con[0] = ovo_f2u(s);
  con[1] = ovo_half_bits_trunc(s) + (ovo_half_bits_trunc(s) << 16); /* AU1_AH2_AF2, ffx_a.h:552 */
  con[2] = 0;
  con[3] = 0;
}

/* PostProcessor.cpp:298-305 (eye 0) and :332-336 (eye 1 when each texture holds one eye).
 * uint*float products are evaluated in float and truncated on assignment to AU1. */
void ovo_centre_radius(uint32_t imageCentre[4], uint32_t radius[4], int eye, int onlyOneEye, uint32_t outW,
                       uint32_t outH, const float proj[4], float radiusCfg) {
  if (eye == 0 || !onlyOneEye) {
    imageCentre[0] = onlyOneEye ? (uint32_t)((float)outW * proj[0]) : (uint32_t)((float)(outW / 2) * proj[0]);
    imageCentre[1] = (uint32_t)((float)outH * proj[1]);
    imageCentre[2] = onlyOneEye ? (uint32_t)((float)outW * proj[0]) : (uint32_t)((float)(outW / 2) * (1 + proj[2]));
    imageCentre[3] = (uint32_t)((float)outH * (onlyOneEye ? proj[1] : proj[3]));
  } else {
    imageCentre[0] = (uint32_t)((float)outW * proj[2]);
    imageCentre[1] = (uint32_t)((float)outH * proj[3]);
    imageCentre[2] = (uint32_t)((float)outW * proj[2]);
    imageCentre[3] = (uint32_t)((float)outH * proj[3]);
  }
  radius[0] = (uint32_t)(0.5f * radiusCfg * (float)outH);
  radius[1] = radius[0] * radius[0]; /* u32 multiply, wraps */
  radius[2] = outW;
  radius[3] = outH;
}

void ovo_make_upscale_constants(ovo_upscale_constants *c, int eye, int onlyOneEye, uint32_t inW, uint32_t inH,
                                uint32_t outW, uint32_t outH, const float proj[4], float radiusCfg) {
  uint32_t con[16];
  /* PostProcessor.cpp:297: viewport == input size */
  ovo_fsr_easu_con(con, (float)inW, (float)inH, (float)inW, (float)inH, (float)outW, (float)outH);
  memcpy(c->const0, con, 16); memcpy(c->const1, con + 4, 16);
  memcpy(c->const2, con + 8, 16); memcpy(c->const3, con + 12, 16);
  ovo_centre_radius(c->imageCentre, c->radius, eye, onlyOneEye, outW, outH, proj, radiusCfg);
}

void ovo_make_sharpen_constants(ovo_sharpen_constants *c, int eye, int onlyOneEye, uint32_t outW, uint32_t outH,
                                const float proj[4], float radiusCfg, float sharpness, int debugMode) {
  /* PostProcessor.cpp:420-421: AClampF1(sharpness,0,1) = max(0,min(s,1)), ffx_a.h:353 */
  float s = sharpness < 1.0f ? sharpness : 1.0f;
  s = 0.0f > s ? 0.0f : s;
  ovo_fsr_rcas_con(c->const0, 2.f - 2 * s);
  ovo_centre_radius(c->imageCentre, c->radius, eye, onlyOneEye, outW, outH, proj, radiusCfg);
  c->const0[3] = debugMode ? 1u : 0u; /* :430 */
}

int ovo_group_inside(uint32_t gx, uint32_t gy, uint32_t gw, uint32_t gh, const uint32_t centre[4], uint32_t radiusSq) {
  return ovo_group_inside_(gx, gy, gw, gh, centre, radiusSq);
}

float ovo_hlsl_min(float a, float b) { return ovo_min(a, b); }
float ovo_hlsl_max(float a, float b) { return ovo_max(a, b); }
float ovo_hlsl_saturate(float a) { return ovo_sat(a); }

/* ------------------------------------------------------------------------
 * approximations, ffx_a.h:1843-1845 (integer bit tricks, portable bit-exactly)
 * ---------------------------------------------------------------------- */
static inline float prx_lo_rcp(float a) { return ovo_u2f(0x7ef07ebbu - ovo_f2u(a)); }
static inline float prx_med_rcp(float a) { float b = ovo_u2f(0x7ef19fffu - ovo_f2u(a)); return b * (-b * a + 2.0f); }
static inline float prx_lo_rsq(float a) { return ovo_u2f(0x5f347d74u - (ovo_f2u(a) >> 1)); }

/* ------------------------------------------------------------------------
 * EASU
 * ---------------------------------------------------------------------- */

/* FsrEasuSetF, ffx_fsr1.h:275-313.  w is the bilinear weight of this corner;
 * (lA..lE) is the '+' of lumas around it:   a / b c d / e. */
static inline void easu_set(float dir[2], float *len, float w, float lA, float lB, float lC, float lD, float lE) {
  float dc = lD - lC, cb = lC - lB;
  float lenX = ovo_max(fabsf(dc), fabsf(cb));
  lenX = prx_lo_rcp(lenX);
  float dirX = lD - lB;
  dir[0] += dirX * w;
  lenX = ovo_sat(fabsf(dirX) * lenX);
  lenX *= lenX;
  *len += lenX * w;
  float ec = lE - lC, ca = lC - lA;
  float lenY = ovo_max(fabsf(ec), fabsf(ca));
  lenY = prx_lo_rcp(lenY);
  float dirY = lE - lA;
  dir[1] += dirY * w;
  lenY = ovo_sat(fabsf(dirY) * lenY);
  lenY *= lenY;
  *len += lenY * w;
}

/* FsrEasuTapF, ffx_fsr1.h:239-272 */
static inline void easu_tap(float aC[3], float *aW, float offX, float offY, const float dir[2], const float len[2],
                            float lob, float clp, const float c[3]) {
  float vx = (offX * (dir[0])) + (offY * dir[1]);
  float vy = (offX * (-dir[1])) + (offY * dir[0]);
  vx *= len[0];
  vy *= len[1];
  float d2 = vx * vx + vy * vy;
  d2 = ovo_min(d2, clp);
  float wB = (float)(2.0 / 5.0) * d2 + (float)(-1.0);
  float wA = lob * d2 + (float)(-1.0);
  wB *= wB;
  wA *= wA;
  wB = (float)(25.0 / 16.0) * wB + (float)(-(25.0 / 16.0 - 1.0));
  float w = wB * wA;
  aC[0] += c[0] * w; aC[1] += c[1] * w; aC[2] += c[2] * w;
  *aW += w;
}

/* FsrEasuF, ffx_fsr1.h:315-437, with the four Gather4 footprints (fsr_easu.hlsl:21-23)
 * expressed as the 12 clamped integer taps they select (SURVEY.md section 8 a4):
 *      b c
 *    e f g h        f = texel (fp.x, fp.y)
 *    i j k l
 *      n o
 */
static void easu_pixel(const ovo_image *src, const ovo_upscale_constants *k, int x, int y, float pix[3]) {
  float ppx = (float)(uint32_t)x * ovo_u2f(k->const0[0]) + ovo_u2f(k->const0[2]);
  float ppy = (float)(uint32_t)y * ovo_u2f(k->const0[1]) + ovo_u2f(k->const0[3]);
  float fpx = floorf(ppx), fpy = floorf(ppy);
  ppx -= fpx;
  ppy -= fpy;
  const int ix = (int)fpx, iy = (int)fpy;

  float b[4], c[4], e[4], f[4], g[4], h[4], i[4], j[4], kk[4], l[4], n[4], o[4];
  ovo_texel_clamp(src, ix + 0, iy - 1, b);
  ovo_texel_clamp(src, ix + 1, iy - 1, c);
  ovo_texel_clamp(src, ix - 1, iy + 0, e);
  ovo_texel_clamp(src, ix + 0, iy + 0, f);
  ovo_texel_clamp(src, ix + 1, iy + 0, g);
  ovo_texel_clamp(src, ix + 2, iy + 0, h);
  ovo_texel_clamp(src, ix - 1, iy + 1, i);
  ovo_texel_clamp(src, ix + 0, iy + 1, j);
  ovo_texel_clamp(src, ix + 1, iy + 1, kk);
  ovo_texel_clamp(src, ix + 2, iy + 1, l);
  ovo_texel_clamp(src, ix + 0, iy + 2, n);
  ovo_texel_clamp(src, ix + 1, iy + 2, o);

  /* luma times 2, :363-366:  B*0.5 + (R*0.5 + G) */
#define LUMA2(t) ((t)[2] * 0.5f + ((t)[0] * 0.5f + (t)[1]))
  const float bL = LUMA2(b), cL = LUMA2(c), eL = LUMA2(e), fL = LUMA2(f), gL = LUMA2(g), hL = LUMA2(h);
  const float iL = LUMA2(i), jL = LUMA2(j), kL = LUMA2(kk), lL = LUMA2(l), nL = LUMA2(n), oL = LUMA2(o);
#undef LUMA2

  /* :380-386 direction and length, bilinear-weighted over the corners f,g,j,k */
  float dir[2] = {0.0f, 0.0f}, len = 0.0f;
  easu_set(dir, &len, (1.0f - ppx) * (1.0f - ppy), bL, eL, fL, gL, jL);
  easu_set(dir, &len, ppx * (1.0f - ppy), cL, fL, gL, hL, kL);
  easu_set(dir, &len, (1.0f - ppx) * ppy, fL, iL, jL, kL, nL);
  easu_set(dir, &len, ppx * ppy, gL, jL, kL, lL, oL);

  /* :389-395 normalise */
  float dir2x = dir[0] * dir[0], dir2y = dir[1] * dir[1];
  float dirR = dir2x + dir2y;
  const int zro = dirR < (float)(1.0 / 32768.0);
  dirR = prx_lo_rsq(dirR);
  dirR = zro ? 1.0f : dirR;
  dir[0] = zro ? 1.0f : dir[0];
  dir[0] *= dirR;
  dir[1] *= dirR;
  /* :397-409 shape */
  len = len * 0.5f;
  len *= len;
  float stretch = (dir[0] * dir[0] + dir[1] * dir[1]) * prx_lo_rcp(ovo_max(fabsf(dir[0]), fabsf(dir[1])));
  float len2[2] = {1.0f + (stretch - 1.0f) * len, 1.0f + (-0.5f) * len};
  float lob = 0.5f + (float)((1.0 / 4.0 - 0.04) - 0.5) * len;
  float clp = prx_lo_rcp(lob);

  /* :416-419 min/max of the 4 nearest (f,g,j,k) */
  float mn4[3], mx4[3];
  for (int ch = 0; ch < 3; ++ch) {
    mn4[ch] = ovo_min(ovo_min(f[ch], ovo_min(g[ch], j[ch])), kk[ch]);
    mx4[ch] = ovo_max(ovo_max(f[ch], ovo_max(g[ch], j[ch])), kk[ch]);
  }

  /* :421-434 accumulate, reference order b c i j f e k l h g o n */
  float aC[3] = {0.0f, 0.0f, 0.0f}, aW = 0.0f;
  easu_tap(aC, &aW, 0.0f - ppx, -1.0f - ppy, dir, len2, lob, clp, b);
  easu_tap(aC, &aW, 1.0f - ppx, -1.0f - ppy, dir, len2, lob, clp, c);
  easu_tap(aC, &aW, -1.0f - ppx, 1.0f - ppy, dir, len2, lob, clp, i);
  easu_tap(aC, &aW, 0.0f - ppx, 1.0f - ppy, dir, len2, lob, clp, j);
  easu_tap(aC, &aW, 0.0f - ppx, 0.0f - ppy, dir, len2, lob, clp, f);
  easu_tap(aC, &aW, -1.0f - ppx, 0.0f - ppy, dir, len2, lob, clp, e);
  easu_tap(aC, &aW, 1.0f - ppx, 1.0f - ppy, dir, len2, lob, clp, kk);
  easu_tap(aC, &aW, 2.0f - ppx, 1.0f - ppy, dir, len2, lob, clp, l);
  easu_tap(aC, &aW, 2.0f - ppx, 0.0f - ppy, dir, len2, lob, clp, h);
  easu_tap(aC, &aW, 1.0f - ppx, 0.0f - ppy, dir, len2, lob, clp, g);
  easu_tap(aC, &aW, 1.0f - ppx, 2.0f - ppy, dir, len2, lob, clp, o);
  easu_tap(aC, &aW, 0.0f - ppx, 2.0f - ppy, dir, len2, lob, clp, n);

  /* :437 normalise and de-ring */
  const float r = rcpf(aW);
  for (int ch = 0; ch < 3; ++ch) pix[ch] = ovo_min(mx4[ch], ovo_max(mn4[ch], aC[ch] * r));
}

/* ------------------------------------------------------------------------
 * RCAS
 * ---------------------------------------------------------------------- */

/* FsrRcasF, ffx_fsr1.h:684-769 with FSR_RCAS_DENOISE and FSR_RCAS_PASSTHROUGH_ALPHA
 * undefined (fsr_rcas.hlsl:1-4), so the nz term (:737-739) is dead and alpha is 1.
 *      b
 *    d e f        Load(): out-of-bounds texels read 0 (fsr_rcas.hlsl:18)
 *      h
 */
static void rcas_pixel(const ovo_image *src, const ovo_sharpen_constants *k, int x, int y, float pix[3]) {
  float b[4], d[4], e[4], f[4], h[4];
  ovo_load(src, x, y - 1, b);
  ovo_load(src, x - 1, y, d);
  ovo_load(src, x, y, e);
  ovo_load(src, x + 1, y, f);
  ovo_load(src, x, y + 1, h);
  float lobeC[3];
  for (int ch = 0; ch < 3; ++ch) {
    /* :741-746 ring min/max: min(AMin3F1(b,d,f),h), AMin3F1(x,y,z)=min(x,min(y,z)) */
    const float mn4 = ovo_min(ovo_min(b[ch], ovo_min(d[ch], f[ch])), h[ch]);
    const float mx4 = ovo_max(ovo_max(b[ch], ovo_max(d[ch], f[ch])), h[ch]);
    /* :748-755 limiters, true reciprocals; peakC = (1.0, -4.0) */
    const float hitMin = mn4 * rcpf(4.0f * mx4);
    const float hitMax = (1.0f - mx4) * rcpf(4.0f * mn4 + (float)(-1.0 * 4.0));
    lobeC[ch] = ovo_max(-hitMin, hitMax); /* :756-758 */
  }
  /* :759  FSR_RCAS_LIMIT = 0.25-1/16, :654 */
  float lobe = ovo_max((float)(-(0.25 - (1.0 / 16.0))),
                       ovo_min(ovo_max(lobeC[0], ovo_max(lobeC[1], lobeC[2])), 0.0f)) *
               ovo_u2f(k->const0[0]);
  /* :765-768 */
  const float rcpL = prx_med_rcp(4.0f * lobe + 1.0f);
  for (int ch = 0; ch < 3; ++ch)
    pix[ch] = (lobe * b[ch] + lobe * d[ch] + lobe * h[ch] + lobe * f[ch] + e[ch]) * rcpL;
}

/* ------------------------------------------------------------------------
 * entry shaders
 * ---------------------------------------------------------------------- */
#define OVO_ENTRY(n) ovo_fsr_##n
#define OVO_EASU_PIXEL(src, c, x, y, o) easu_pixel(src, c, x, y, o)
#define OVO_RCAS_PIXEL(src, c, x, y, o) rcas_pixel(src, c, x, y, o)
#include "fsr_entry.inc"

int ovo_fsr_easu(const ovo_image *src, const ovo_image *dst, const ovo_upscale_constants *c, int nthreads) {
  return ovo_fsr_run_easu(src, dst, c, nthreads);
}
int ovo_fsr_rcas(const ovo_image *src, const ovo_image *dst, const ovo_sharpen_constants *c, int nthreads) {
  return ovo_fsr_run_rcas(src, dst, c, nthreads);
}

/*
 * cas_oracle.c -- CPU restatement of the legacy FidelityFX CAS path of openvr_fsr (src/cas; SURVEY.md 8f row 4).
 *
 * TEST INFRASTRUCTURE ONLY: the checker for the CUDA CAS kernels; only tests/ may link or load it.
 * The reference never dispatches these shaders (src/CMakeLists.txt compiles only fsr/ and nis/), so "the reference
 * result" is what its source says: src/cas/cas.compute.h (entry), src/cas/ffx_cas.h:375-397 (CasSetup) and :409-893
 * (CasFilter, the non-packed float path: A_HLSL without A_HALF, so CAS_GO_SLOWER and CAS_SLOW are undefined and the
 * bit-trick approximations APrxLoRcpF1 / APrxLoSqrtF1 / APrxMedRcpF1 of src/cas/ffx_a.h:1455-1457 apply).
 * Pinned against those very lines compiled on the host: oracle/_ref (ref_shim/cas_ref.cpp), tests/test_cas.py.
 *
 * Arithmetic is binary32 in the reference's operation order, no contraction (-ffp-contract=off); min/max ignore NaN;
 * CasLoad = Texture2D.Load (0 outside the image).  Only the green weights are live: with CAS_SLOW undefined the
 * red / blue amplitude chains feed nothing (ffx_cas.h:514-523,869-878).
 */
#include <math.h>

#include "ovr_oracle.h"
#include "ovr_glue.h"

static inline float mn2(float a, float b) { return ovo_min(a, b); }
static inline float mx2(float a, float b) { return ovo_max(a, b); }
static inline float mn3(float x, float y, float z) { return mn2(x, mn2(y, z)); } /* AMin3F1 */
static inline float mx3(float x, float y, float z) { return mx2(x, mx2(y, z)); } /* AMax3F1 */
static inline float prx_lo_rcp(float a) { return ovo_u2f(0x7ef07ebbu - ovo_f2u(a)); }
static inline float prx_lo_sqrt(float a) { return ovo_u2f((ovo_f2u(a) >> 1) + 0x1fbc4639u); }
static inline float prx_med_rcp(float a) { float b = ovo_u2f(0x7ef19fffu - ovo_f2u(a)); return b * (-b * a + 2.0f); }

/* ffx_cas.h:375-397 with the A_CPU helpers of src/cas/ffx_a.h (ALerpF1 :302, ASatF1 :366, ARcpF1 :330) */
void ovo_cas_setup(ovo_cas_constants *c, float sharpness, float maxColorDelta, float inW, float inH, float outW, float outH) {
  c->const0[0] = ovo_f2u(inW * (1.0f / outW));
  c->const0[1] = ovo_f2u(inH * (1.0f / outH));
  c->const0[2] = ovo_f2u(0.5f * inW * (1.0f / outW) - 0.5f);
  c->const0[3] = ovo_f2u(0.5f * inH * (1.0f / outH) - 0.5f);
  const float s = (0.0f > sharpness) ? 0.0f : sharpness, t = (1.0f < s) ? 1.0f : s; /* AMinF1(1, AMaxF1(0, x)) */
  const float lerp = 5.0f * t + (-8.0f * t + 8.0f);                                   /* ALerpF1(8,5,t) = b*c+(-a*c+a) */
  const float sharp = -(1.0f / lerp);
  c->const1[0] = ovo_f2u(sharp);
  c->const1[1] = ovo_half_bits_trunc(sharp) + (ovo_half_bits_trunc(maxColorDelta) << 16);
  c->const1[2] = ovo_f2u(8.0f * inW * (1.0f / outW));
  c->const1[3] = ovo_f2u(maxColorDelta);
}

static inline void ld(const ovo_image *im, int x, int y, float o[3]) {
  float t[4];
  ovo_load(im, x, y, t);
  o[0] = t[0]; o[1] = t[1]; o[2] = t[2];
}

/* sharpen-only branch with CAS_BETTER_DIAGONALS, ffx_cas.h:424-551 */
static void cas_sharpen_px(const ovo_image *src, const ovo_cas_constants *k, int x, int y, float o[4]) {
  float a[3], b[3], c[3], d[3], e[3], f[3], g[3], h[3], i[3];
  ld(src, x - 1, y - 1, a); ld(src, x, y - 1, b); ld(src, x + 1, y - 1, c);
  ld(src, x - 1, y, d);     ld(src, x, y, e);     ld(src, x + 1, y, f);
  ld(src, x - 1, y + 1, g); ld(src, x, y + 1, h); ld(src, x + 1, y + 1, i);
  /* soft min / max of the green channel: cross, then cross + diagonals, summed */
  float mn = mn3(mn3(d[1], e[1], f[1]), b[1], h[1]);
  const float mnD = mn3(mn3(mn, a[1], c[1]), g[1], i[1]);
  mn = mn + mnD;
  float mx = mx3(mx3(d[1], e[1], f[1]), b[1], h[1]);
  const float mxD = mx3(mx3(mx, a[1], c[1]), g[1], i[1]);
  mx = mx + mxD;
  float amp = ovo_sat(mn2(mn, 2.0f - mx) * prx_lo_rcp(mx));
  amp = prx_lo_sqrt(amp);
  const float w = amp * ovo_u2f(k->const1[0]);
  const float rcpW = prx_med_rcp(1.0f + 4.0f * w);
  const float mcd = ovo_u2f(k->const1[3]);
  for (int ch = 0; ch < 3; ++ch) {
    const float p = ovo_sat((b[ch] * w + d[ch] * w + f[ch] * w + h[ch] * w + e[ch]) * rcpW);
    o[ch] = mn2(mx2(p, e[ch] - mcd), e[ch] + mcd); /* clamp(pix, e-maxColorDelta, e+maxColorDelta) */
  }
}

/* green soft-min/max of the '+' around (x,y): up, left, centre, right, down -- ffx_cas.h:610-706 without diagonals */
static inline void plus_mn_mx(const ovo_image *src, int x, int y, float *mn, float *mx) {
  float u[3], l[3], c[3], r[3], d[3];
  ld(src, x, y - 1, u); ld(src, x - 1, y, l); ld(src, x, y, c); ld(src, x + 1, y, r); ld(src, x, y + 1, d);
  *mn = mn3(mn3(u[1], l[1], c[1]), r[1], d[1]);
  *mx = mx3(mx3(u[1], l[1], c[1]), r[1], d[1]);
}

/* scaling branch, ffx_cas.h:553-893 (cas.upscale.hlsl: no CAS_BETTER_DIAGONALS) */
static void cas_scale_px(const ovo_image *src, const ovo_cas_constants *k, int x, int y, float o[4]) {
  float ppx = (float)(uint32_t)x * ovo_u2f(k->const0[0]) + ovo_u2f(k->const0[2]);
  float ppy = (float)(uint32_t)y * ovo_u2f(k->const0[1]) + ovo_u2f(k->const0[3]);
  const float fx = floorf(ppx), fy = floorf(ppy);
  ppx -= fx; ppy -= fy;
  const int sx = (int)fx, sy = (int)fy;
  /*  a b c d / e f g h / i j k l / m n o p ; a, d, m, p are fetched by the shader but feed nothing here */
  float b[3], c[3], e[3], f[3], g[3], h[3], i[3], j[3], kk[3], l[3], n[3], oo[3];
  ld(src, sx, sy - 1, b);     ld(src, sx + 1, sy - 1, c);
  ld(src, sx - 1, sy, e);     ld(src, sx, sy, f);         ld(src, sx + 1, sy, g);     ld(src, sx + 2, sy, h);
  ld(src, sx - 1, sy + 1, i); ld(src, sx, sy + 1, j);     ld(src, sx + 1, sy + 1, kk); ld(src, sx + 2, sy + 1, l);
  ld(src, sx, sy + 2, n);     ld(src, sx + 1, sy + 2, oo);
  float mnf, mxf, mng, mxg, mnj, mxj, mnk, mxk;
  plus_mn_mx(src, sx, sy, &mnf, &mxf);
  plus_mn_mx(src, sx + 1, sy, &mng, &mxg);
  plus_mn_mx(src, sx, sy + 1, &mnj, &mxj);
  plus_mn_mx(src, sx + 1, sy + 1, &mnk, &mxk);
  const float peak = ovo_u2f(k->const1[0]);
  const float wf = prx_lo_sqrt(ovo_sat(mn2(mnf, 1.0f - mxf) * prx_lo_rcp(mxf))) * peak;
  const float wg = prx_lo_sqrt(ovo_sat(mn2(mng, 1.0f - mxg) * prx_lo_rcp(mxg))) * peak;
  const float wj = prx_lo_sqrt(ovo_sat(mn2(mnj, 1.0f - mxj) * prx_lo_rcp(mxj))) * peak;
  const float wk = prx_lo_sqrt(ovo_sat(mn2(mnk, 1.0f - mxk) * prx_lo_rcp(mxk))) * peak;
  float s = (1.0f - ppx) * (1.0f - ppy), t = ppx * (1.0f - ppy), u = (1.0f - ppx) * ppy, v = ppx * ppy;
  const float thinB = 1.0f / 32.0f;
  s *= prx_lo_rcp(thinB + (mxf - mnf));
  t *= prx_lo_rcp(thinB + (mxg - mng));
  u *= prx_lo_rcp(thinB + (mxj - mnj));
  v *= prx_lo_rcp(thinB + (mxk - mnk));
  const float qbe = wf * s, qch = wg * t;
  const float qf = wg * t + wj * u + s, qg = wf * s + wk * v + t, qj = wf * s + wk * v + u, qk = wg * t + wj * u + v;
  const float qin = wj * u, qlo = wk * v;
  const float rcpW = prx_med_rcp(2.0f * qbe + 2.0f * qch + 2.0f * qin + 2.0f * qlo + qf + qg + qj + qk);
  for (int ch = 0; ch < 3; ++ch)
    o[ch] = ovo_sat((b[ch] * qbe + e[ch] * qbe + c[ch] * qch + h[ch] * qch + i[ch] * qin + n[ch] * qin + l[ch] * qlo +
                     oo[ch] * qlo + f[ch] * qf + g[ch] * qg + j[ch] * qj + kk[ch] * qk) * rcpW);
}

static inline void cas_px(const ovo_image *src, const ovo_cas_constants *k, int sharpen_only, int x, int y, float o[4]) {
  if (sharpen_only) cas_sharpen_px(src, k, x, y, o);
  else cas_scale_px(src, k, x, y, o);
}

#define OVO_ENTRY(n) ovo_cas_##n
#define OVO_CAS_PIXEL(src, c, so, x, y, o) cas_px(src, c, so, x, y, o)
#include "cas_entry.inc"

int ovo_cas(const ovo_image *src, const ovo_image *dst, const ovo_cas_constants *c, int sharpen_only, int nthreads) {
  if (sharpen_only && src && dst && (src->width != dst->width || src->height != dst->height)) return -1;
  return ovo_cas_run_cas(src, dst, c, sharpen_only, nthreads);
}

/*
 * nis_oracle.c -- CPU restatement of the NVIDIA Image Scaling half of the openvr_fsr hot path: NISConfig
 * setup, NVScaler (directional 6-tap scale + sharpen) and NVSharpen (directional USM), stated per OUTPUT
 * PIXEL.  The reference evaluates the same functions through a group-shared luma / edge-map tile
 * (src/nis/NIS_Scaler.h:310-316,613-673); the tile is only a cache of per-source-texel values, so the
 * per-pixel statement below yields identical bits, which tests/test_oracle_vs_ref.py checks against the
 * reference header compiled verbatim (oracle/_ref).
 *
 * TEST INFRASTRUCTURE ONLY -- see ovr_oracle.h.  Build: gcc -O2 -ffp-contract=off.
 * Citations: /root/reference/src/nis/.  lerp(x,y,s) = x + s*(y-x); a/b is IEEE division.
 */
#include "ovr_glue.h"

#include "nis_coef.inc"

static float g_scale[64][8], g_usm[64][8];
static int g_coef_ready = 0;
static void coef_init(void) {
  if (g_coef_ready) return;
  for (int p = 0; p < 64; ++p)
    for (int t = 0; t < 8; ++t) {
      g_scale[p][t] = t < 6 ? (float)(kNisCoefScale1e4[p][t] / 10000.0) : 0.0f;
      g_usm[p][t] = t < 6 ? (float)(kNisCoefUsm1e4[p][t] / 10000.0) : 0.0f;
    }
  __sync_synchronize();
  g_coef_ready = 1;
}
const float *ovo_nis_coef_scale(void) { coef_init(); return &g_scale[0][0]; }
const float *ovo_nis_coef_usm(void) { coef_init(); return &g_usm[0][0]; }

/* NVScalerUpdateConfig, NIS_Config.h:144-241 (SDR branch), argument pattern of PostProcessor.cpp:308/433 */
static int nis_update(ovo_nis_config *c, float sharpness, uint32_t inW, uint32_t inH, uint32_t outW, uint32_t outH) {
  memset(c, 0, sizeof(*c));
  sharpness = ovo_max(ovo_min(1.f, sharpness), 0.f);
  const float slider = sharpness - 0.5f;
  const float MinScale = (slider >= 0.0f) ? 1.25f : 1.0f;
  const float LimitScale = (slider >= 0.0f) ? 1.25f : 1.0f;
  const float kMinContrastRatio = 2.0f, kMaxContrastRatio = 10.0f, kSharpStartY = 0.45f, kSharpEndY = 0.9f;
  const float kSharpStrengthMin = ovo_max(0.0f, 0.4f + slider * MinScale * 1.2f);
  const float kSharpStrengthMax = 1.6f + slider * 1.8f;
  const float kSharpLimitMin = ovo_max(0.1f, 0.14f + slider * LimitScale * 0.32f);
  const float kSharpLimitMax = 0.5f + slider * LimitScale * 0.6f;
  c->kInputViewportWidth = inW; c->kInputViewportHeight = inH;
  c->kOutputViewportWidth = outW; c->kOutputViewportHeight = outH;
  if (!inW || !inH || !outW || !outH) return 0;
  c->kSrcNormX = 1.f / inW; c->kSrcNormY = 1.f / inH;
  c->kDstNormX = 1.f / outW; c->kDstNormY = 1.f / outH;
  c->kScaleX = inW / (float)outW;
  c->kScaleY = inH / (float)outH;
  if (c->kScaleX < 0.5f || c->kScaleX > 1.f || c->kScaleY < 0.5f || c->kScaleY > 1.f) return 0;
  c->kDetectRatio = 1127.f / 1024.f;
  c->kDetectThres = 64.0f / 1024.0f;
  c->kMinContrastRatio = kMinContrastRatio;
  c->kRatioNorm = 1.0f / (kMaxContrastRatio - kMinContrastRatio);
  c->kContrastBoost = 1.0f;
  c->kEps = 1.0f;
  c->kSharpStartY = kSharpStartY;
  c->kSharpScaleY = 1.0f / (kSharpEndY - kSharpStartY);
  c->kSharpStrengthMin = kSharpStrengthMin;
  c->kSharpStrengthScale = kSharpStrengthMax - kSharpStrengthMin;
  c->kSharpLimitMin = kSharpLimitMin;
  c->kSharpLimitScale = kSharpLimitMax - kSharpLimitMin;
  return 1;
}

int ovo_make_nis_config(ovo_nis_config *c, int sharpenOnly, int eye, int onlyOneEye, uint32_t inW, uint32_t inH,
                        uint32_t outW, uint32_t outH, const float proj[4], float radiusCfg, float sharpness,
                        int debugMode) {
  const int ok = sharpenOnly ? nis_update(c, sharpness, inW, inH, inW, inH) : nis_update(c, sharpness, inW, inH, outW, outH);
  c->reserved1 = debugMode ? 1.f : 0.f;                                                  /* PostProcessor.cpp:309 */
  ovo_centre_radius(c->imageCentre, c->radius, eye, onlyOneEye, outW, outH, proj, radiusCfg); /* :310 memcpy */
  return ok;
}

/* ---- shared pieces ------------------------------------------------------------------------------------ */
static inline float lerpf(float x, float y, float s) { return x + s * (y - x); }

/* getY, NIS_Scaler.h:160-169 (NIS_HDR_MODE_NONE) on a clamped texel: what a linear-clamp SampleLevel aimed at a
 * texel centre returns (NIS_Scaler.h:634-651,893-900) */
static inline float luma_at(const ovo_image *src, int x, int y) {
  float t[4];
  ovo_texel_clamp(src, x, y, t);
  return 0.2126f * t[0] + 0.7152f * t[1] + 0.0722f * t[2];
}

/* GetEdgeMap, NIS_Scaler.h:176-293, on the 3x3 luma window w[row][col] (luma in [0,1] units) */
static void edge_map(const ovo_nis_config *k, float w[3][3], float out[4]) {
  const float g_0 = fabsf(w[0][0] + w[0][1] + w[0][2] - w[2][0] - w[2][1] - w[2][2]);
  const float g_45 = fabsf(w[1][0] + w[0][0] + w[0][1] - w[2][1] - w[2][2] - w[1][2]);
  const float g_90 = fabsf(w[0][0] + w[1][0] + w[2][0] - w[0][2] - w[1][2] - w[2][2]);
  const float g_135 = fabsf(w[1][0] + w[2][0] + w[2][1] - w[0][1] - w[0][2] - w[1][2]);
  const float g_0_90_max = ovo_max(g_0, g_90), g_0_90_min = ovo_min(g_0, g_90);
  const float g_45_135_max = ovo_max(g_45, g_135), g_45_135_min = ovo_min(g_45, g_135);
  float e_0_90 = 0, e_45_135 = 0;
  if ((g_0_90_max + g_45_135_max) != 0) {
    e_0_90 = g_0_90_max / (g_0_90_max + g_45_135_max);
    e_0_90 = ovo_min(e_0_90, 1.0f);
    e_45_135 = 1.0f - e_0_90;
  }
  float edge_0 = 0, edge_45 = 0, edge_90 = 0, edge_135 = 0;
  if ((g_0_90_max > (g_0_90_min * k->kDetectRatio)) && (g_0_90_max > k->kDetectThres) && (g_0_90_max > g_45_135_min)) {
    if (g_0_90_max == g_0) edge_0 = 1.0f; else edge_90 = 1.0f;
  }
  if ((g_45_135_max > (g_45_135_min * k->kDetectRatio)) && (g_45_135_max > k->kDetectThres) && (g_45_135_max > g_0_90_min)) {
    if (g_45_135_max == g_45) edge_45 = 1.0f; else edge_135 = 1.0f;
  }
  const float nEdges = edge_0 + edge_90 + edge_45 + edge_135;
  if (nEdges >= 2.0f) {
    out[0] = (edge_0 == 1.0f) ? e_0_90 : 0;  out[1] = (edge_0 == 1.0f) ? 0 : e_0_90;
    out[2] = (edge_45 == 1.0f) ? e_45_135 : 0; out[3] = (edge_45 == 1.0f) ? 0 : e_45_135;
  } else if (nEdges >= 1.0f) {
    out[0] = edge_0; out[1] = edge_90; out[2] = edge_45; out[3] = edge_135;
  } else {
    out[0] = out[1] = out[2] = out[3] = 0;
  }
}

static void edge_map_at(const ovo_image *src, const ovo_nis_config *k, int x, int y, float out[4]) {
  float w[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) w[r][c] = luma_at(src, x - 1 + c, y - 1 + r);
  edge_map(k, w, out);
}

/* the contrast-ratio term shared by CalcLTI (:343-375) and CalcLTIFast (:790-803) */
static inline float lti(const ovo_nis_config *k, float y0, float y1, float y2, float y3, float y4, float eps) {
  const float a_min = ovo_min(ovo_min(y0, y1), y2), a_max = ovo_max(ovo_max(y0, y1), y2);
  const float b_min = ovo_min(ovo_min(y2, y3), y4), b_max = ovo_max(ovo_max(y2, y3), y4);
  const float a_cont = a_max - a_min, b_cont = b_max - b_min;
  const float cont_ratio = ovo_max(a_cont, b_cont) / (ovo_min(a_cont, b_cont) + eps);
  return (1.0f - ovo_sat((cont_ratio - k->kMinContrastRatio) * k->kRatioNorm)) * k->kContrastBoost;
}

/* ---- NVScaler -------------------------------------------------------------------------------------------- */
/* EvalPoly6, NIS_Scaler.h:399-434: 6-tap polyphase scale + luma-adaptive USM with anti-ringing */
static float eval_poly6(const ovo_nis_config *k, const float pxl[6], int phase) {
  float y = 0.f, y_usm = 0.f;
  for (int i = 0; i < 6; ++i) y += g_scale[phase][i] * pxl[i];
  for (int i = 0; i < 6; ++i) y_usm += g_usm[phase][i] * pxl[i];
  const float y_scale = 1.0f - ovo_sat((y * (1.0f / 255) - k->kSharpStartY) * k->kSharpScaleY);
  const float y_sharpness = y_scale * k->kSharpStrengthScale + k->kSharpStrengthMin;
  y_usm *= y_sharpness;
  const float y_sharpness_limit = (y_scale * k->kSharpLimitScale + k->kSharpLimitMin) * y;
  y_usm = ovo_min(y_sharpness_limit, ovo_max(-y_sharpness_limit, y_usm));
  /* CalcLTI: phases <= 32 look at taps 0..4, later phases at taps 1..5 */
  const int o = phase <= 64 / 2 ? 0 : 1;
  y_usm *= lti(k, pxl[o], pxl[o + 1], pxl[o + 2], pxl[o + 3], pxl[o + 4], k->kEps);
  return y + y_usm;
}

/* FilterNormal, NIS_Scaler.h:436-453: separable 6x6, columns first */
static float filter_normal(float p[6][6], int phx, int phy) {
  float h_acc = 0.0f;
  for (int j = 0; j < 6; ++j) {
    float v_acc = 0.0f;
    for (int i = 0; i < 6; ++i) v_acc += p[i][j] * g_scale[phy][i];
    h_acc += v_acc * g_scale[phx][j];
  }
  return h_acc;
}

/* GetDirFilters, NIS_Scaler.h:455-583: the 0 / 90 / 45 / 135 degree 6-tap lines through the 6x6 window */
static void dir_filters(const ovo_nis_config *k, float p[6][6], float fx, float fy, int phx, int phy, float f[4]) {
  float line[6];
  for (int i = 0; i < 6; ++i) line[i] = lerpf(p[i][2], p[i][3], fx);
  f[0] = eval_poly6(k, line, phy);
  for (int i = 0; i < 6; ++i) line[i] = lerpf(p[2][i], p[3][i], fy);
  f[1] = eval_poly6(k, line, phx);

  /* 45 degrees (:482-528) */
  float b45 = 0.5f + 0.5f * (fx - fy);
  float t[7];
  t[1] = lerpf(p[2][1], p[1][2], b45);
  t[3] = lerpf(p[3][2], p[2][3], b45);
  t[5] = lerpf(p[4][3], p[3][4], b45);
  if (b45 >= 0.5f) {
    b45 = b45 - 0.5f;
    t[0] = lerpf(p[1][1], p[0][2], b45);
    t[2] = lerpf(p[2][2], p[1][3], b45);
    t[4] = lerpf(p[3][3], p[2][4], b45);
    t[6] = lerpf(p[4][4], p[3][5], b45);
  } else {
    b45 = 0.5f - b45;
    t[0] = lerpf(p[1][1], p[2][0], b45);
    t[2] = lerpf(p[2][2], p[3][1], b45);
    t[4] = lerpf(p[3][3], p[4][2], b45);
    t[6] = lerpf(p[4][4], p[5][3], b45);
  }
  float p45 = fx + fy;
  int sh = 0;
  if (p45 >= 1) { sh = 1; p45 = p45 - 1; }
  for (int i = 0; i < 6; ++i) line[i] = t[i + sh];
  f[2] = eval_poly6(k, line, (int)(p45 * 64));

  /* 135 degrees (:530-581) */
  float b135 = 0.5f * (fx + fy);
  t[1] = lerpf(p[3][1], p[4][2], b135);
  t[3] = lerpf(p[2][2], p[3][3], b135);
  t[5] = lerpf(p[1][3], p[2][4], b135);
  if (b135 >= 0.5f) {
    b135 = b135 - 0.5f;
    t[0] = lerpf(p[4][1], p[5][2], b135);
    t[2] = lerpf(p[3][2], p[4][3], b135);
    t[4] = lerpf(p[2][3], p[3][4], b135);
    t[6] = lerpf(p[1][4], p[2][5], b135);
  } else {
    b135 = 0.5f - b135;
    t[0] = lerpf(p[4][1], p[3][0], b135);
    t[2] = lerpf(p[3][2], p[2][1], b135);
    t[4] = lerpf(p[2][3], p[1][2], b135);
    t[6] = lerpf(p[1][4], p[0][3], b135);
  }
  float p135 = 1 + (fx - fy);
  sh = 0;
  if (p135 >= 1) { sh = 1; p135 = p135 - 1; }
  for (int i = 0; i < 6; ++i) line[i] = t[i + sh];
  f[3] = eval_poly6(k, line, (int)(p135 * 64));
}

/* NVScaler's per-pixel phase, NIS_Scaler.h:675-769 */
static void nis_scaler_pixel(const ovo_image *src, const ovo_nis_config *k, int dstX, int dstY, float op[4]) {
  const float srcX = (0.5f + dstX) * k->kScaleX - 0.5f;
  const float srcY = (0.5f + dstY) * k->kScaleY - 0.5f;
  const int x0 = (int)floorf(srcX), y0 = (int)floorf(srcY);
  /* 6x6 luma support around floor(src), scaled to 0..255 as the shared tile stores it (:664-668) */
  float p[6][6];
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) p[i][j] = luma_at(src, x0 - 2 + j, y0 - 2 + i) * 255.0f;
  const float fx = srcX - floorf(srcX), fy = srcY - floorf(srcY);
  const int fx_int = (int)(fx * 64), fy_int = (int)(fy * 64);
  const float pixel_n = filter_normal(p, fx_int, fy_int);
  float d[4];
  dir_filters(k, p, fx, fy, fx_int, fy_int, d);
  /* 2x2 edge maps centred in the window, bilinearly interpolated (:727-738, GetInterpEdgeMap :377-397) */
  float e[2][2][4], w[4];
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) edge_map_at(src, k, x0 + j, y0 + i, e[i][j]);
  for (int c = 0; c < 4; ++c) {
    const float h0 = lerpf(e[0][0][c], e[0][1][c], fx), h1 = lerpf(e[1][0][c], e[1][1][c], fx);
    w[c] = lerpf(h0, h1, fy) * 255.0f; /* * NIS_SCALE_INT */
  }
  const float opY = (d[0] * w[0] + d[1] * w[1] + d[2] * w[2] + d[3] * w[3] +
                     pixel_n * (255.0f - w[0] - w[1] - w[2] - w[3])) * (1.0f / 255.0f);
  /* one bilinear RGBA tap for chroma, then add the luma correction (:747-761); alpha is the sampled alpha */
  ovo_sample_linear(src, (dstX + 0.5f) * k->kDstNormX, (dstY + 0.5f) * k->kDstNormY, op);
  const float corr = opY * (1.0f / 255.0f) - (0.2126f * op[0] + 0.7152f * op[1] + 0.0722f * op[2]);
  op[0] += corr; op[1] += corr; op[2] += corr;
}

/* ---- NVSharpen ------------------------------------------------------------------------------------------- */
/* EvalUSM, NIS_Scaler.h:805-817 */
static float eval_usm(const ovo_nis_config *k, const float pxl[5], float strength, float limit) {
  float y_usm = -0.6001f * pxl[1] + 1.2002f * pxl[2] - 0.6001f * pxl[3];
  y_usm *= strength;
  y_usm = ovo_min(limit, ovo_max(-limit, y_usm));
  y_usm *= lti(k, pxl[0], pxl[1], pxl[2], pxl[3], pxl[4], k->kEps * (1.0f / 255.0f)); /* CalcLTIFast */
  return y_usm;
}

/* NVSharpen's per-pixel phase, NIS_Scaler.h:905-969 with GetDirUSM :819-871 */
static void nis_sharpen_pixel(const ovo_image *src, const ovo_nis_config *k, int dstX, int dstY, float op[4]) {
  float p[5][5];
  for (int i = 0; i < 5; ++i)
    for (int j = 0; j < 5; ++j) p[i][j] = luma_at(src, dstX - 2 + j, dstY - 2 + i);
  const float scaleY = 1.0f - ovo_sat((p[2][2] - k->kSharpStartY) * k->kSharpScaleY);
  const float strength = scaleY * k->kSharpStrengthScale + k->kSharpStrengthMin;
  const float limit = (scaleY * k->kSharpLimitScale + k->kSharpLimitMin) * p[2][2];
  float line[5], u[4];
  for (int i = 0; i < 5; ++i) line[i] = p[i][2];
  u[0] = eval_usm(k, line, strength, limit);
  for (int i = 0; i < 5; ++i) line[i] = p[2][i];
  u[1] = eval_usm(k, line, strength, limit);
  line[0] = p[1][1]; line[1] = lerpf(p[2][1], p[1][2], 0.5f); line[2] = p[2][2];
  line[3] = lerpf(p[3][2], p[2][3], 0.5f); line[4] = p[3][3];
  u[2] = eval_usm(k, line, strength, limit);
  line[0] = p[3][1]; line[1] = lerpf(p[3][2], p[2][1], 0.5f); line[2] = p[2][2];
  line[3] = lerpf(p[2][3], p[1][2], 0.5f); line[4] = p[1][3];
  u[3] = eval_usm(k, line, strength, limit);
  float w3[3][3], w[4];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) w3[r][c] = p[1 + r][1 + c]; /* GetEdgeMap(p, 1, 1) */
  edge_map(k, w3, w);
  const float usmY = (u[0] * w[0] + u[1] * w[1] + u[2] * w[2] + u[3] * w[3]);
  ovo_sample_linear(src, (dstX + 0.5f) * k->kDstNormX, (dstY + 0.5f) * k->kDstNormY, op);
  op[0] += usmY; op[1] += usmY; op[2] += usmY;
}

/* ---- entry shaders ---------------------------------------------------------------------------------------- */
static void scaler_block(const ovo_image *src, const ovo_image *dst, const ovo_nis_config *k, uint32_t bx, uint32_t by) {
  for (int py = 0; py < 24; ++py)
    for (int px = 0; px < 32; ++px) {
      const int x = (int)bx * 32 + px, y = (int)by * 24 + py;
      if (x >= dst->width || y >= dst->height) continue;
      float op[4];
      nis_scaler_pixel(src, k, x, y, op);
      ovo_store(dst, x, y, op);
    }
}
static void sharpen_block(const ovo_image *src, const ovo_image *dst, const ovo_nis_config *k, uint32_t bx, uint32_t by) {
  for (int py = 0; py < 32; ++py)
    for (int px = 0; px < 32; ++px) {
      const int x = (int)bx * 32 + px, y = (int)by * 32 + py;
      if (x >= dst->width || y >= dst->height) continue;
      float op[4];
      nis_sharpen_pixel(src, k, x, y, op);
      ovo_store(dst, x, y, op);
    }
}

#define OVO_ENTRY(n) ovo_nis_scaler_##n
#define OVO_NIS_IS_SHARPEN 0
#define OVO_NIS_BIND(src, dst, cfg) coef_init()
#define OVO_NIS_BLOCK(src, dst, cfg, bx, by) scaler_block(src, dst, cfg, bx, by)
#include "nis_entry.inc"
#undef OVO_ENTRY
#undef OVO_NIS_IS_SHARPEN
#undef OVO_NIS_BIND
#undef OVO_NIS_BLOCK

#define OVO_ENTRY(n) ovo_nis_sharpen_##n
#define OVO_NIS_IS_SHARPEN 1
#define OVO_NIS_BIND(src, dst, cfg) (void)0
#define OVO_NIS_BLOCK(src, dst, cfg, bx, by) sharpen_block(src, dst, cfg, bx, by)
#include "nis_entry.inc"

int ovo_nis_scaler(const ovo_image *src, const ovo_image *dst, const ovo_nis_config *c, int nthreads) {
  coef_init();
  return ovo_nis_scaler_run(src, dst, c, nthreads);
}
int ovo_nis_sharpen(const ovo_image *src, const ovo_image *dst, const ovo_nis_config *c, int nthreads) {
  return ovo_nis_sharpen_run(src, dst, c, nthreads);
}

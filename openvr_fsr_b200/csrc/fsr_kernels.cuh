// fsr_kernels.cuh -- FSR1 EASU (upscale) and RCAS (sharpen) for sm_90a.
//
// Replaces the two D3D11 compute dispatches of the reference:
//   g_FSRUpscaleShader = src/fsr/fsr_easu.hlsl:38-64 -> FsrEasuF, src/fsr/ffx_fsr1.h:315-437
//   g_FSRSharpenShader = src/fsr/fsr_rcas.hlsl:29-55 -> FsrRcasF, src/fsr/ffx_fsr1.h:684-769
// (citations relative to /root/reference/).  Not a translation of the HLSL: the work is
// re-tiled for a CTA of 8 warps over a 64x32 output tile,
//   * the source tile (+halo) is decoded ONCE per texel into shared memory (float4 rgb + luma);
//     the reference decodes every texel ~21 times through 36 Gather4s per pixel,
//   * EASU's direction/length analysis (FsrEasuSetF) depends only on the '+' neighbourhood of a
//     SOURCE texel, so it is evaluated once per source texel into a shared feature tile and
//     each output pixel bilinearly blends four float4 features instead of redoing 4 x ~25 ops,
//   * one warp owns one 16x16 output group, so the reference's per-workgroup radius test is a
//     warp-uniform branch (no divergence) with the bilinear / copy fast path fused in.
// Arithmetic order inside each reference function is kept where kStrict is set, so the strict
// build is bit-identical to the reference lines; the fast build regroups the 12 tap offsets
// (v = A*o - A*pp for integer o) and lets ptxas contract FMAs.
#pragma once

#include "device_common.cuh"
#include "tma_utils.cuh"

namespace ovrfsr {
inline namespace OVRFSR_MODE_NS {

constexpr int kTileW = 64;   // output tile of one CTA
constexpr int kTileH = 32;
constexpr int kThreads = 256; // 8 warps, one per 16x16 group

struct EasuArgs {
  ImageRO src;
  ImageRW dst;
  float c0x, c0y, c0z, c0w; // const0 of FsrEasuCon: out->in scale and offset
  uint32_t centre[4];
  uint32_t radiusSq;
  float radW, radH;         // (float)Radius.z, (float)Radius.w for Bilinear()
  int tileW, tileH;         // shared source tile extent in texels
  // When RCAS follows in the same apply (ctx path only): outside-radius groups are final after this pass -- RCAS would
  // only copy them (x the debug tint) -- so they are written straight to the final image `direct`, and to the
  // intermediate `dst` only where an edge-adjacent group is inside the radius (RCAS reads one pixel across the edge).
  ImageRW direct;           // ptr == nullptr: plain dispatch
  float tintGB;             // 1 - debug*0.3 of the following RCAS pass
};

struct RcasArgs {
  ImageRO src;
  ImageRW dst;
  float sharp;              // const0[0] as float
  float tintGB;             // 1 - debug*0.3 (fsr_rcas.hlsl:46)
  uint32_t centre[4];
  uint32_t radiusSq;
  int skipOutside;          // the preceding EASU launch already wrote the outside-radius groups to dst (EasuArgs::direct)
  int opaqueSrc;            // B8G8R8X8 source: the X byte reads as alpha 1 (only the outside-radius copy looks at alpha)
};

// out pixel -> source position; the same instruction sequence is used for the tile origin and
// for every pixel so that both agree to the bit.
__device__ __forceinline__ float easu_pos(int p, float scale, float offs) { return mul_add_unfused((float)p, scale, offs); }

// FsrEasuSetF (ffx_fsr1.h:275-313) minus the bilinear weight: the per-source-texel part.
//   a
// b c d      returns (dirX, dirY, lenX, lenY)
//   e
__device__ __forceinline__ float4 easu_feature(float lA, float lB, float lC, float lD, float lE) {
  const float dc = lD - lC, cb = lC - lB;
  float lenX = prx_lo_rcp(fmaxf(fabsf(dc), fabsf(cb)));
  const float dirX = lD - lB;
  lenX = __saturatef(fabsf(dirX) * lenX);
  lenX *= lenX;
  const float ec = lE - lC, ca = lC - lA;
  float lenY = prx_lo_rcp(fmaxf(fabsf(ec), fabsf(ca)));
  const float dirY = lE - lA;
  lenY = __saturatef(fabsf(dirY) * lenY);
  lenY *= lenY;
  return make_float4(dirX, dirY, lenX, lenY);
}

// ---- strict math: FsrEasuF in the reference's operation order (scalar) ----------------------------------------
// Products the reference recomputes per tap are formed once: off.x*dir.x and off.x*(-dir.y) for the 4 distinct
// off.x, off.y*dir.y and off.y*dir.x for the 4 distinct off.y -- same operands, same product, 16 multiplies
// instead of 48.
// FsrEasuTapF, ffx_fsr1.h:239-272, from the two products of each coordinate
__device__ __forceinline__ void easu_tap_ref(float &aR, float &aG, float &aB, float &aW, float xdx, float ydy, float xndy,
                                             float ydx, float len0, float len1, float lob, float clp, const float4 c) {
  float vx = xdx + ydy;   // (off.x*dir.x) + (off.y*dir.y)
  float vy = xndy + ydx;  // (off.x*(-dir.y)) + (off.y*dir.x)
  vx *= len0;
  vy *= len1;
  float d2 = vx * vx + vy * vy;
  d2 = fminf(d2, clp);
  float wB = (float)(2.0 / 5.0) * d2 + (float)(-1.0);
  float wA = lob * d2 + (float)(-1.0);
  wB *= wB;
  wA *= wA;
  wB = (float)(25.0 / 16.0) * wB + (float)(-(25.0 / 16.0 - 1.0));
  const float w = wB * wA;
  aR += c.x * w; aG += c.y * w; aB += c.z * w;
  aW += w;
}

// FsrEasuF, ffx_fsr1.h:315-437, for the output pixel whose 'f' texel is cf in the colour tile and fr in the feature
// tile, with sub-texel phase (ppx,ppy) >= +0.
//
// Two kinds of reference additions are left out, because they can only change the sign of a zero that is then
// squared:
//  * the zero the feature sums start from (0 + p = p except p = -0).  Each len term is lenX or lenY (saturated, >= +0)
//    times a bilinear weight (>= +0), never -0, so len has the same bits.  dirX / dirY can differ only in the sign of a
//    zero.  After the normalisation (x dirR > 0, or 1 when both are below 1/32768) they reach the output only through
//    squares, fabsf, and the products off*dir.  Those products are summed into vx / vy, which differ at most in the
//    sign of a zero and are squared into d2.  A NaN or inf operand gives the same NaN either way.
//  * 0 - pp for the tap offset 0: -pp differs only for pp = +0, and then off*dir is a zero that feeds vx / vy as above.
// The colour and weight sums still start from zero: their sign can reach the output.
template <int TW>
__device__ __forceinline__ float3 easu_filter(const float4 *__restrict__ cf, const float4 *__restrict__ fr, float ppx,
                                              float ppy) {
  // direction + length: bilinear blend of the four corner features (:380-386)
  const float4 Ff = fr[0], Fg = fr[1], Fj = fr[TW], Fk = fr[TW + 1];
  const float qx = 1.0f - ppx, qy = 1.0f - ppy;
  const float wf = qx * qy, wg = ppx * qy, wj = qx * ppy, wk = ppx * ppy;
  float dirX = Ff.x * wf, len = Ff.z * wf, dirY = Ff.y * wf;
  len += Ff.w * wf;
  dirX += Fg.x * wg; len += Fg.z * wg; dirY += Fg.y * wg; len += Fg.w * wg;
  dirX += Fj.x * wj; len += Fj.z * wj; dirY += Fj.y * wj; len += Fj.w * wj;
  dirX += Fk.x * wk; len += Fk.z * wk; dirY += Fk.y * wk; len += Fk.w * wk;

  // normalise (:389-395)
  const float dir2x = dirX * dirX, dir2y = dirY * dirY;
  float dirR = dir2x + dir2y;
  const bool zro = dirR < (float)(1.0 / 32768.0);
  dirR = prx_lo_rsq(dirR);
  dirR = zro ? 1.0f : dirR;
  dirX = zro ? 1.0f : dirX;
  dirX *= dirR;
  dirY *= dirR;
  // shape (:397-409)
  len = len * 0.5f;
  len *= len;
  const float stretch = (dirX * dirX + dirY * dirY) * prx_lo_rcp(fmaxf(fabsf(dirX), fabsf(dirY)));
  const float len0 = 1.0f + (stretch - 1.0f) * len;
  const float len1 = 1.0f + (-0.5f) * len;
  const float lob = 0.5f + (float)((1.0 / 4.0 - 0.04) - 0.5) * len;
  const float clp = prx_lo_rcp(lob);

  // the 4 distinct off.x / off.y values and their products with dir (shared by the 12 taps)
  const float ndirY = -dirY;
  const float ox0 = -1.0f - ppx, ox1 = -ppx, ox2 = 1.0f - ppx, ox3 = 2.0f - ppx;
  const float oy0 = -1.0f - ppy, oy1 = -ppy, oy2 = 1.0f - ppy, oy3 = 2.0f - ppy;
  const float xd0 = ox0 * dirX, xd1 = ox1 * dirX, xd2 = ox2 * dirX, xd3 = ox3 * dirX;
  const float xn0 = ox0 * ndirY, xn1 = ox1 * ndirY, xn2 = ox2 * ndirY, xn3 = ox3 * ndirY;
  const float yd0 = oy0 * dirY, yd1 = oy1 * dirY, yd2 = oy2 * dirY, yd3 = oy3 * dirY;
  const float yx0 = oy0 * dirX, yx1 = oy1 * dirX, yx2 = oy2 * dirX, yx3 = oy3 * dirX;

  //    b c
  //  e f g h
  //  i j k l
  //    n o
  const float4 *r0 = cf - TW;
  const float4 f = r0[TW], g = r0[TW + 1], j = r0[2 * TW], k = r0[2 * TW + 1];
  float aR = 0.0f, aG = 0.0f, aB = 0.0f, aW = 0.0f;
  // reference accumulation order (:423-434): b c i j f e k l h g o n   (index 0..3 <-> offset -1..2)
  easu_tap_ref(aR, aG, aB, aW, xd1, yd0, xn1, yx0, len0, len1, lob, clp, r0[0]);          // b ( 0,-1)
  easu_tap_ref(aR, aG, aB, aW, xd2, yd0, xn2, yx0, len0, len1, lob, clp, r0[1]);          // c ( 1,-1)
  easu_tap_ref(aR, aG, aB, aW, xd0, yd2, xn0, yx2, len0, len1, lob, clp, r0[2 * TW - 1]); // i (-1, 1)
  easu_tap_ref(aR, aG, aB, aW, xd1, yd2, xn1, yx2, len0, len1, lob, clp, j);              // j ( 0, 1)
  easu_tap_ref(aR, aG, aB, aW, xd1, yd1, xn1, yx1, len0, len1, lob, clp, f);              // f ( 0, 0)
  easu_tap_ref(aR, aG, aB, aW, xd0, yd1, xn0, yx1, len0, len1, lob, clp, r0[TW - 1]);     // e (-1, 0)
  easu_tap_ref(aR, aG, aB, aW, xd2, yd2, xn2, yx2, len0, len1, lob, clp, k);              // k ( 1, 1)
  easu_tap_ref(aR, aG, aB, aW, xd3, yd2, xn3, yx2, len0, len1, lob, clp, r0[2 * TW + 2]); // l ( 2, 1)
  easu_tap_ref(aR, aG, aB, aW, xd3, yd1, xn3, yx1, len0, len1, lob, clp, r0[TW + 2]);     // h ( 2, 0)
  easu_tap_ref(aR, aG, aB, aW, xd2, yd1, xn2, yx1, len0, len1, lob, clp, g);              // g ( 1, 0)
  easu_tap_ref(aR, aG, aB, aW, xd2, yd3, xn2, yx3, len0, len1, lob, clp, r0[3 * TW + 1]); // o ( 1, 2)
  easu_tap_ref(aR, aG, aB, aW, xd1, yd3, xn1, yx3, len0, len1, lob, clp, r0[3 * TW]);     // n ( 0, 2)

  // min/max of the four nearest (:416-419), normalise and de-ring (:437)
  const float mnR = fminf(fminf(f.x, fminf(g.x, j.x)), k.x), mxR = fmaxf(fmaxf(f.x, fmaxf(g.x, j.x)), k.x);
  const float mnG = fminf(fminf(f.y, fminf(g.y, j.y)), k.y), mxG = fmaxf(fmaxf(f.y, fmaxf(g.y, j.y)), k.y);
  const float mnB = fminf(fminf(f.z, fminf(g.z, j.z)), k.z), mxB = fmaxf(fmaxf(f.z, fmaxf(g.z, j.z)), k.z);
  const float r = rcp_mode(aW);
  return make_float3(fminf(mxR, fmaxf(mnR, aR * r)), fminf(mxG, fmaxf(mnG, aG * r)), fminf(mxB, fmaxf(mnB, aB * r)));
}

// ---- fast math: FsrEasuF regrouped in two-lane (f2) form ------------------------------------------------------
// Same function as easu_filter, evaluated differently (results differ from the reference lines in the last
// bits only; <= 1 LSB after RGBA8 rounding):
//   * the squared rotated/stretched tap distance is a quadratic form of the integer tap offset,
//       d2(ox,oy) = Q00*dx^2 + 2*Q01*dx*dy + Q11*dy^2,  dx = ox-ppx, dy = oy-ppy,  Q = M^T M,
//     so one add2 + one fma2 yield d2 for two horizontally adjacent taps (A_P + B_j, E_P*dy_j);
//   * the window polynomial is expanded: 25/16*(2/5 t-1)^2 - 9/16 = (t/4 - 5/4) t + 1;
//   * the colour tile stores (r,g,b,1): two fma2 per tap accumulate (r,g) and (b, weight) at once;
//   * feature blending, normalisation and setup are grouped the same way.
__device__ __forceinline__ f2 easu_w2(f2 A, float B, f2 E, float dy, float clp, float lob) {
  f2 t = fma2(E, bc(dy), add2(A, bc(B)));
  t.x = fminf(t.x, clp);
  t.y = fminf(t.y, clp);
  const f2 base = fma2(fma2(t, bc(0.25f), bc(-1.25f)), t, bc(1.0f));
  f2 win = fma2(t, bc(lob), bc(-1.0f));
  win = mul2(win, win);
  return mul2(base, win);
}
__device__ __forceinline__ void easu_acc(f2 &aRG, f2 &aBW, const float4 c, float w) {
  aRG = fma2(make_float2(c.x, c.y), bc(w), aRG);
  aBW = fma2(make_float2(c.z, c.w), bc(w), aBW); // c.w == 1: the weight sum rides along
}

template <int TW>
__device__ __forceinline__ float3 easu_filter_fast(const float4 *__restrict__ cf, const float4 *__restrict__ fr, float ppx,
                                                   float ppy) {
  const float4 Ff = fr[0], Fg = fr[1], Fj = fr[TW], Fk = fr[TW + 1];
  const float qx = 1.0f - ppx, qy = 1.0f - ppy;
  const f2 wt = mul2(make_float2(qx, ppx), bc(qy)), wb = mul2(make_float2(qx, ppx), bc(ppy)); // (wf,wg) (wj,wk)
  f2 dir = mul2(make_float2(Ff.x, Ff.y), bc(wt.x));
  f2 ln = mul2(make_float2(Ff.z, Ff.w), bc(wt.x));
  dir = fma2(make_float2(Fg.x, Fg.y), bc(wt.y), dir); ln = fma2(make_float2(Fg.z, Fg.w), bc(wt.y), ln);
  dir = fma2(make_float2(Fj.x, Fj.y), bc(wb.x), dir); ln = fma2(make_float2(Fj.z, Fj.w), bc(wb.x), ln);
  dir = fma2(make_float2(Fk.x, Fk.y), bc(wb.y), dir); ln = fma2(make_float2(Fk.z, Fk.w), bc(wb.y), ln);
  float len = ln.x + ln.y;

  f2 dd = mul2(dir, dir);
  float dirR = dd.x + dd.y;
  const bool zro = dirR < (float)(1.0 / 32768.0);
  dirR = zro ? 1.0f : prx_lo_rsq(dirR);
  dir.x = zro ? 1.0f : dir.x;
  dir = mul2(dir, bc(dirR));
  len = len * 0.5f;
  len *= len;
  dd = mul2(dir, dir);
  const float stretch = (dd.x + dd.y) * prx_lo_rcp(fmaxf(fabsf(dir.x), fabsf(dir.y)));
  const float len0 = fmaf(stretch - 1.0f, len, 1.0f);
  const float len1 = fmaf(-0.5f, len, 1.0f);
  const float lob = fmaf((float)((1.0 / 4.0 - 0.04) - 0.5), len, 0.5f);
  const float clp = prx_lo_rcp(lob);

  // Q = M^T M with M = diag(len0,len1) * Rot(dir):  Q00 = dx^2 L0 + dy^2 L1, Q11 = dy^2 L0 + dx^2 L1, Q01 = dx dy (L0-L1)
  const float L0 = len0 * len0, L1 = len1 * len1;
  const float Q00 = fmaf(dd.x, L0, dd.y * L1), Q11 = fmaf(dd.y, L0, dd.x * L1);
  const float Q01x2 = 2.0f * (dir.x * dir.y) * (L0 - L1);
  // tap offsets: x pairs (-1,0) (0,1) (1,2), y scalars -1,0,1,2
  const f2 mpx = bc(-ppx), mpy = bc(-ppy);
  const f2 dxA = add2(make_float2(-1.0f, 0.0f), mpx), dxB = add2(make_float2(0.0f, 1.0f), mpx),
           dxC = add2(make_float2(1.0f, 2.0f), mpx);
  const f2 dyA = add2(make_float2(-1.0f, 0.0f), mpy), dyB = add2(make_float2(1.0f, 2.0f), mpy);
  const f2 qq = bc(Q00), ee = bc(Q01x2), q11 = bc(Q11);
  const f2 AA = mul2(mul2(dxA, dxA), qq), AB = mul2(mul2(dxB, dxB), qq), AC = mul2(mul2(dxC, dxC), qq);
  const f2 EA = mul2(dxA, ee), EB = mul2(dxB, ee), EC = mul2(dxC, ee);
  const f2 BA = mul2(mul2(dyA, dyA), q11), BB = mul2(mul2(dyB, dyB), q11); // (B_-1,B_0) (B_1,B_2)

  //    b c
  //  e f g h
  //  i j k l
  //    n o
  const float4 *r0 = cf - TW;
  f2 aRG = bc(0.0f), aBW = bc(0.0f);
  {
    const float4 b = r0[0], c = r0[1];
    const f2 w = easu_w2(AB, BA.x, EB, dyA.x, clp, lob);
    easu_acc(aRG, aBW, b, w.x); easu_acc(aRG, aBW, c, w.y);
  }
  const float4 f = r0[TW], g = r0[TW + 1], j = r0[2 * TW], k = r0[2 * TW + 1];
  {
    const float4 e = r0[TW - 1], h = r0[TW + 2];
    const f2 w0 = easu_w2(AA, BA.y, EA, dyA.y, clp, lob), w1 = easu_w2(AC, BA.y, EC, dyA.y, clp, lob);
    easu_acc(aRG, aBW, e, w0.x); easu_acc(aRG, aBW, f, w0.y);
    easu_acc(aRG, aBW, g, w1.x); easu_acc(aRG, aBW, h, w1.y);
  }
  {
    const float4 i = r0[2 * TW - 1], l = r0[2 * TW + 2];
    const f2 w0 = easu_w2(AA, BB.x, EA, dyB.x, clp, lob), w1 = easu_w2(AC, BB.x, EC, dyB.x, clp, lob);
    easu_acc(aRG, aBW, i, w0.x); easu_acc(aRG, aBW, j, w0.y);
    easu_acc(aRG, aBW, k, w1.x); easu_acc(aRG, aBW, l, w1.y);
  }
  {
    const float4 n = r0[3 * TW], o = r0[3 * TW + 1];
    const f2 w = easu_w2(AB, BB.y, EB, dyB.y, clp, lob);
    easu_acc(aRG, aBW, n, w.x); easu_acc(aRG, aBW, o, w.y);
  }
  const float mnR = fminf(fminf(f.x, fminf(g.x, j.x)), k.x), mxR = fmaxf(fmaxf(f.x, fmaxf(g.x, j.x)), k.x);
  const float mnG = fminf(fminf(f.y, fminf(g.y, j.y)), k.y), mxG = fmaxf(fmaxf(f.y, fmaxf(g.y, j.y)), k.y);
  const float mnB = fminf(fminf(f.z, fminf(g.z, j.z)), k.z), mxB = fmaxf(fmaxf(f.z, fmaxf(g.z, j.z)), k.z);
  const float r = rcp_mode(aBW.y);
  return make_float3(fminf(mxR, fmaxf(mnR, aRG.x * r)), fminf(mxG, fmaxf(mnG, aRG.y * r)), fminf(mxB, fmaxf(mnB, aBW.x * r)));
}

// Bilinear(), fsr_easu.hlsl:33-36: SampleLevel(linearClamp, float2(pos)/Radius.zw) -- no half-texel
// offset; coordinates snapped to 1/256 texel like D3D11's fixed-point sampler.  The sample position is separable:
// the x part (one IEEE divide, snap, floor) depends only on the output column and the y part only on the output row,
// so each is evaluated once per column / row instead of once per pixel -- same operations, same bits.
struct BilinAxis { int t0, t1; float f; }; // clamped tile coordinates of the two taps and the weight of the second
__device__ __forceinline__ BilinAxis easu_bilinear_axis(int p, float rad, int srcExtent, int tileOrigin, int tileExtent) {
  const float u = (float)p / rad;
  const float s = snap_subtexel(mul_add_unfused(u, (float)srcExtent, -0.5f));
  const float s0 = floorf(s);
  BilinAxis r;
  r.f = s - s0;
  r.t0 = clampi((int)s0 - tileOrigin, 0, tileExtent - 1);
  r.t1 = clampi((int)s0 + 1 - tileOrigin, 0, tileExtent - 1);
  return r;
}
__device__ __forceinline__ float3 easu_bilinear(const float4 *__restrict__ sC, int tw, const BilinAxis ax, const BilinAxis ay) {
  const float4 c00 = sC[ay.t0 * tw + ax.t0], c10 = sC[ay.t0 * tw + ax.t1];
  const float4 c01 = sC[ay.t1 * tw + ax.t0], c11 = sC[ay.t1 * tw + ax.t1];
  const float fx = ax.f, fy = ay.f, wx0 = 1.0f - fx, wy0 = 1.0f - fy;
  const float tR = c00.x * wx0 + c10.x * fx, bR = c01.x * wx0 + c11.x * fx;
  const float tG = c00.y * wx0 + c10.y * fx, bG = c01.y * wx0 + c11.y * fx;
  const float tB = c00.z * wx0 + c10.z * fx, bB = c01.z * wx0 + c11.z * fx;
  return make_float3(tR * wy0 + bR * fy, tG * wy0 + bG * fy, tB * wy0 + bB * fy);
}

// 3-channel decode of a packed RGBA8/BGRA8 texel (EASU never reads source alpha: its output alpha is 1).
// ALWAYS the exact decode, also in fast math: where luma is flat but chroma varies, FsrEasuSetF divides rounding
// noise by rounding noise (|lD-lB| / max(|lD-lC|,|lC-lB|) with all three lumas equal up to the last bit), so the
// edge strength there is defined by the exact bits of the decoded values; a decode that is 1 ulp off changes the
// result by several LSB at such pixels.
template <int FMT>
__device__ __forceinline__ float4 decode_rgb1(uint32_t p) {
  if constexpr (FMT == OVRFSR_FORMAT_RGB10A2) return make_float4(unorm10(p & 1023u), unorm10((p >> 10) & 1023u), unorm10((p >> 20) & 1023u), 1.0f);
  const float c0 = unorm8(byte_to_float<0>(p)), c1 = unorm8(byte_to_float<1>(p)), c2 = unorm8(byte_to_float<2>(p));
  if constexpr (FMT == OVRFSR_FORMAT_BGRA8) return make_float4(c2, c1, c0, 1.0f);
  return make_float4(c0, c1, c2, 1.0f);
}
template <int FMT>
__device__ __forceinline__ float4 decode_rgba(uint32_t p) {
  if constexpr (FMT == OVRFSR_FORMAT_RGB10A2) return decode_rgb10a2(p);
  const float c0 = byte_to_unorm_mode<0>(p), c1 = byte_to_unorm_mode<1>(p);
  const float c2 = byte_to_unorm_mode<2>(p), c3 = byte_to_unorm_mode<3>(p);
  if constexpr (FMT == OVRFSR_FORMAT_BGRA8) return make_float4(c2, c1, c0, c3);
  return make_float4(c0, c1, c2, c3);
}

// FLOAT -> intermediate UNORM -> FLOAT, the store / Load round trip of the two-dispatch form
template <int FMID>
__device__ __forceinline__ float4 mid_roundtrip(float r, float g, float b) {
  if constexpr (FMID == OVRFSR_FORMAT_RGB10A2) {
    return make_float4(unorm10(to_unorm<1023>(r)), unorm10(to_unorm<1023>(g)), unorm10(to_unorm<1023>(b)), 1.0f);
  } else {
    // to_unorm8 then the decode rcas_kernel applies to an RGBA8 source (decode_rgba: exact in strict math, the
    // single-FFMA form in fast math); the code is already an integer, so 2^23 + v is one LOP3 instead of a PRMT
    const uint32_t cr = to_unorm8(r) | 0x4B000000u, cg = to_unorm8(g) | 0x4B000000u, cb = to_unorm8(b) | 0x4B000000u;
    if constexpr (kStrict) {
      return make_float4(unorm8(u2f(cr) - 8388608.0f), unorm8(u2f(cg) - 8388608.0f), unorm8(u2f(cb) - 8388608.0f), 1.0f);
    } else {
      const float k = 1.0f / 255.0f;
      return make_float4(__fmaf_rn(u2f(cr), k, -8388608.0f * k), __fmaf_rn(u2f(cg), k, -8388608.0f * k),
                         __fmaf_rn(u2f(cb), k, -8388608.0f * k), 1.0f);
    }
  }
}

// One-colour groups.  FsrEasuF ends in the de-ring clamp min(mx, max(mn, aC*rcp(aW))) with mn / mx over the four
// nearest texels f, g, j, k.  Where those four have the same RGB, mn == mx == f and the clamp returns f whatever the
// taps summed to: a finite v gives max(f, v) >= f and then min(f, .) == f, a NaN gives f (min / max ignore NaN).  A
// decoded UNORM texel is a finite value >= +0 (no -0, no NaN), so such a pixel is exactly encode(f), in both math modes.
// The footprint of a group -- every f / g / j / k any of its in-image pixels uses -- is the texel rectangle
// floor(pos(first)) .. floor(pos(last)) + 1 in each axis (easu_pos is monotone).  Returns the tile offset of its first
// texel when the whole rectangle has one RGB, else -1.  Tile coordinates: the tile is already clamped to the image edge.
// Called by all 32 lanes of a warp: 16 columns x 2 rows per step, leaving at the first step that finds a second colour.
template <int TW>
__device__ __forceinline__ int easu_flat_group(const float4 *__restrict__ sC, const EasuArgs &a, int lane, int gx, int gy,
                                               int tx0, int sy0) {
  const int fx0 = (int)floorf(easu_pos(gx, a.c0x, a.c0z)) - tx0;
  const int fx1 = (int)floorf(easu_pos(min(gx + 15, a.dst.w - 1), a.c0x, a.c0z)) + 1 - tx0;
  const int fy0 = (int)floorf(easu_pos(gy, a.c0y, a.c0w)) - sy0;
  const int fy1 = (int)floorf(easu_pos(min(gy + 15, a.dst.h - 1), a.c0y, a.c0w)) + 1 - sy0;
  const float4 ref = sC[fy0 * TW + fx0];
  for (int r = fy0; r <= fy1; r += 2) {
    const int ty = r + (lane >> 4);
    bool same = true;
    for (int c = fx0; c <= fx1; c += 16) {
      const int tx = c + (lane & 15);
      if (ty <= fy1 && tx <= fx1) {
        const float4 t = sC[ty * TW + tx];
        same = same && f2u(t.x) == f2u(ref.x) && f2u(t.y) == f2u(ref.y) && f2u(t.z) == f2u(ref.z);
      }
    }
    if (!__all_sync(0xFFFFFFFFu, same)) return -1;
  }
  return fy0 * TW + fx0;
}

// TW  = shared tile row stride in texels (compile time, so every tap is base + immediate): 60 covers out->in
//       scales up to 0.81 for a 64-wide output tile (60 texels incl. the 4 TMA alignment columns), 72 the rest up to 1.0.
// TMA = the raw RGBA8 source box (tile + halo) arrives by cp.async.bulk.tensor into a landing zone and is decoded
//       from there; otherwise (FP16/FP32 sources, unaligned pitch) texels are fetched with plain loads.
constexpr int kEasuRowsPerThread = 5;  // tile rows handled by one warp: ceil(37 / 8)
constexpr int kEasuColsPerThread = 3;  // 32-wide column blocks: ceil(72 / 32)

// PAIRED = RCAS follows in the same apply (EasuArgs::direct is set): a compile-time variant, so that the plain dispatch
// keeps exactly the instruction stream it had without the pairing.
// ANYIO = any of src (TMA == false only), dst and direct may be a CUDA array (`io`); otherwise `io` is unused.
template <int FIN, int FOUT, int TW, bool TMA, bool PAIRED, bool ANYIO>
__global__ void __launch_bounds__(kThreads, 3) easu_kernel(const __grid_constant__ EasuArgs a,
                                                           const __grid_constant__ CUtensorMap srcMap,
                                                           const __grid_constant__ ArrayIO io) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  __shared__ uint64_t tileBar;
  __shared__ BilinAxis sRowAxis[kTileH]; // Bilinear()'s row terms of this tile (outside-radius groups only)
  const int th = a.tileH, tn = TW * th;
  float4 *sC = reinterpret_cast<float4 *>(smem_raw);  // decoded colour (r,g,b,1)
  float4 *sF = sC + tn;                               // (dirX, dirY, lenX, lenY) per texel
  float *sL = reinterpret_cast<float *>(sF + tn);     // luma*2 plane (conflict-free stencil reads)
  const int rawW = a.tileW + 4;                       // TMA box width (origin floored to 4 texels)
  uint32_t *sRaw = reinterpret_cast<uint32_t *>(smem_raw + ((tn * 36 + 127) & ~127)); // landing zone (TMA only), 128-byte aligned

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // One 64x32 output tile per CTA, handed to the SMs by the hardware block scheduler: a tile costs what its content
  // asks for (one-colour groups skip the filter, see easu_flat_group), so a static walk over the tiles would leave
  // the SMs with the most filtered groups finishing last.
  const int ox0 = blockIdx.x * kTileW, oy0 = blockIdx.y * kTileH;
  // source tile origin: one texel left/above the 'f' texel of the tile's first pixel
  const int sx0 = (int)floorf(easu_pos(ox0, a.c0x, a.c0z)) - 1;
  const int sy0 = (int)floorf(easu_pos(oy0, a.c0y, a.c0w)) - 1;
  if constexpr (TMA) {
    if (tid == 0) {
      mbar_init(&tileBar, 1);
      fence_barrier_init();
      mbar_arrive_expect_tx(&tileBar, (uint32_t)(rawW * th * 4));
      tma_load_2d(sRaw, &srcMap, sx0 & ~3, sy0, &tileBar); // box origin 16-byte aligned in x
    }
    __syncthreads();
  }

  // float-tile origin and width in source texels: the TMA variant keeps the box's aligned origin
  const int tx0 = TMA ? (sx0 & ~3) : sx0;
  const int cols = TMA ? rawW : a.tileW;

  // this warp's 16x16 group and its radius test (warp-uniform)
  const uint32_t ggx = (uint32_t)(ox0 >> 4) + (warp & 3), ggy = (uint32_t)(oy0 >> 4) + (warp >> 2);
  const bool inside = group_inside(ggx * 16u + 8u, ggy * 16u + 8u, a.centre, a.radiusSq);

  // ---- stage 1: decode the clamped source tile once, loads batched per thread for ILP -------------
  if constexpr (TMA) {
    mbar_wait(&tileBar, 0); // the tile's box has landed (zeros outside the image)
    const uint32_t *raw = sRaw;
#pragma unroll
    for (int i = 0; i < kEasuColsPerThread; ++i) {
      const int tx = lane + 32 * i;
      if (tx < cols) {
        const int rcol = clampi(tx0 + tx, 0, a.src.w - 1) - tx0; // clamp-to-edge: re-read the edge column / row
        uint32_t px[kEasuRowsPerThread];
#pragma unroll
        for (int j = 0; j < kEasuRowsPerThread; ++j) {
          const int ty = warp + 8 * j;
          px[j] = ty < th ? raw[(clampi(sy0 + ty, 0, a.src.h - 1) - sy0) * rawW + rcol] : 0u;
        }
#pragma unroll
        for (int j = 0; j < kEasuRowsPerThread; ++j) {
          const int ty = warp + 8 * j;
          if (ty < th) {
            const float4 c = decode_rgb1<FIN>(px[j]);
            sL[ty * TW + tx] = c.z * 0.5f + (c.x * 0.5f + c.y); // luma*2, ffx_fsr1.h:363 (x0.5 exact: FMA-safe)
            sC[ty * TW + tx] = c;
          }
        }
      }
    }
  } else {
    // plain loads (FP16 / FP32 sources, unaligned pitch): a flat index over the tile, four texels per thread in
    // flight (no prefetch hides this latency, unlike the TMA variant)
    const int nTex = cols * th;
    const uint32_t colsRcp = 0xFFFFFFFFu / (uint32_t)cols + 1u; // ceil(2^32 / cols): q / cols == umulhi(q, colsRcp) for q < 2^32 / cols
#pragma unroll 4
    for (int q = tid; q < nTex; q += kThreads) {
      const int ty = (int)__umulhi((uint32_t)q, colsRcp), tx = q - ty * cols;
      const int gy = clampi(sy0 + ty, 0, a.src.h - 1), gx = clampi(tx0 + tx, 0, a.src.w - 1);
      float4 c = get_texel<FIN, ANYIO>(a.src, io.src, gx, gy);
      sL[ty * TW + tx] = c.z * 0.5f + (c.x * 0.5f + c.y);
      c.w = 1.0f; // EASU ignores source alpha; the fast path accumulates the tap weight through this lane
      sC[ty * TW + tx] = c;
    }
  }
  // one row term per output row of the tile for the bilinear fallback (skipped when every group is inside)
  if (tid < kTileH && oy0 + tid < a.dst.h) sRowAxis[tid] = easu_bilinear_axis(oy0 + tid, a.radH, a.src.h, sy0, th);
  // inside groups whose footprint has one colour store f and need neither the filter nor the features (UNORM
  // sources only: a float source can hold -0 and NaN, for which the argument at easu_flat_group does not hold).
  // The skip is decided here, per group, never at launch: which kernel a dispatch launches depends on formats and
  // layouts only, not on texel values (tests/test_gpu_float_signed.py relies on that for its coverage count).
  int flatAt = -1;
  if constexpr (packed32(FIN)) {
    __syncthreads();
    if (inside) flatAt = easu_flat_group<TW>(sC, a, lane, (int)ggx * 16, (int)ggy * 16, tx0, sy0);
  }
  const int anyFilter = __syncthreads_or(inside && flatAt < 0);

  // ---- stage 2: per-source-texel direction/length features (only where EASU will run) -----------
  if (anyFilter) {
#pragma unroll
    for (int i = 0; i < kEasuColsPerThread; ++i) {
      const int tx = 1 + lane + 32 * i;
      if (tx < cols - 1) {
        float lA[kEasuRowsPerThread], lB[kEasuRowsPerThread], lC[kEasuRowsPerThread], lD[kEasuRowsPerThread],
            lE[kEasuRowsPerThread];
#pragma unroll
        for (int j = 0; j < kEasuRowsPerThread; ++j) {
          const int ty = 1 + warp + 8 * j;
          if (ty < th - 1) {
            const float *l = sL + ty * TW + tx;
            lA[j] = l[-TW]; lB[j] = l[-1]; lC[j] = l[0]; lD[j] = l[1]; lE[j] = l[TW];
          }
        }
#pragma unroll
        for (int j = 0; j < kEasuRowsPerThread; ++j) {
          const int ty = 1 + warp + 8 * j;
          if (ty < th - 1) sF[ty * TW + tx] = easu_feature(lA[j], lB[j], lC[j], lD[j], lE[j]);
        }
      }
    }
    __syncthreads();
  }

  // ---- stage 3: one warp per 16x16 group, 8 pixels per lane --------------------------------------
  const int x = (int)ggx * 16 + (lane & 15);
  if (x < a.dst.w) {
    const int yFirst = (int)ggy * 16 + (lane >> 4);
    if (inside && flatAt >= 0) {
      const float4 f = sC[flatAt];
      if constexpr (ANYIO) {
        for (int y = yFirst; y < a.dst.h && y < yFirst + 16; y += 2) put_opaque<FOUT, ANYIO>(a.dst, io.dst, x, y, f.x, f.y, f.z);
      } else {
        const texel_t<FOUT> v = encode_opaque<FOUT>(f.x, f.y, f.z);
        uint8_t *out = a.dst.ptr + (size_t)yFirst * a.dst.pitch + (size_t)x * sizeof(texel_t<FOUT>);
        for (int y = yFirst; y < a.dst.h && y < yFirst + 16; y += 2) {
          *reinterpret_cast<texel_t<FOUT> *>(out) = v;
          out += 2 * (size_t)a.dst.pitch;
        }
      }
    } else if (inside) {
      const float ppx_full = easu_pos(x, a.c0x, a.c0z);
      const float fpx = floorf(ppx_full);
      const float ppx = ppx_full - fpx;
      const int ix = (int)fpx - tx0 - sy0 * TW; // tile offset of texel (fpx, 0)
      const int yEnd = min(yFirst + 16, a.dst.h);
      // pitched target: the store address advances by two rows per pixel instead of being formed from (x, y)
      uint8_t *out = a.dst.ptr + (size_t)yFirst * a.dst.pitch + (size_t)x * sizeof(texel_t<FOUT>);
#pragma unroll 2
      for (int y = yFirst; y < yEnd; y += 2) {
        const float ppy_full = easu_pos(y, a.c0y, a.c0w);
        const float fpy = floorf(ppy_full);
        const int o = (int)fpy * TW + ix;
        float3 c;
        if constexpr (kStrict) c = easu_filter<TW>(sC + o, sF + o, ppx, ppy_full - fpy);
        else c = easu_filter_fast<TW>(sC + o, sF + o, ppx, ppy_full - fpy);
        if constexpr (ANYIO) {
          put_opaque<FOUT, ANYIO>(a.dst, io.dst, x, y, c.x, c.y, c.z);
        } else {
          *reinterpret_cast<texel_t<FOUT> *>(out) = encode_opaque<FOUT>(c.x, c.y, c.z);
          out += 2 * (size_t)a.dst.pitch;
        }
      }
    } else {
      const BilinAxis ax = easu_bilinear_axis(x, a.radW, a.src.w, tx0, cols);
      constexpr bool direct = PAIRED && (FOUT == OVRFSR_FORMAT_RGBA8 || FOUT == OVRFSR_FORMAT_RGB10A2);
      // the intermediate is still needed where RCAS of an edge-adjacent inside group reads across the group edge
      const bool mid = !direct || group_inside(ggx * 16u - 8u, ggy * 16u + 8u, a.centre, a.radiusSq) ||
                       group_inside(ggx * 16u + 24u, ggy * 16u + 8u, a.centre, a.radiusSq) ||
                       group_inside(ggx * 16u + 8u, ggy * 16u - 8u, a.centre, a.radiusSq) ||
                       group_inside(ggx * 16u + 8u, ggy * 16u + 24u, a.centre, a.radiusSq);
#pragma unroll 2
      for (int k = 0; k < 8; ++k) {
        const int y = yFirst + 2 * k;
        if (y >= a.dst.h) break;
        const float3 c = easu_bilinear(sC, TW, ax, sRowAxis[y - oy0]);
        if (mid) put_opaque<FOUT, ANYIO>(a.dst, io.dst, x, y, c.x, c.y, c.z);
        if constexpr (direct) {
          if (a.tintGB == 1.0f) {
            // RCAS's copy is the identity on UNORM codes (decode -> x1 -> encode): the same bits go to the final image
            put_opaque<FOUT, ANYIO>(a.direct, io.direct, x, y, c.x, c.y, c.z);
          } else {
            // OutputTexture[p] = mul * InputTexture[p] on the stored-then-loaded value (fsr_rcas.hlsl:45-53)
            const float4 m = mid_roundtrip<FOUT>(c.x, c.y, c.z);
            put_texel<FOUT, ANYIO>(a.direct, io.direct, x, y, 1.0f * m.x, a.tintGB * m.y, a.tintGB * m.z, 1.0f * m.w);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// RCAS
// ------------------------------------------------------------------------------------------------
constexpr int kRcasTW = kTileW + 4;  // float tile: 1-texel halo each side, padded to a multiple of 4 texels
constexpr int kRcasTH = kTileH + 2;
constexpr int kRcasRawW = kTileW + 8; // TMA box: starts 4 texels left of the tile (16-byte aligned origin), 1 used right

// FsrRcasF, ffx_fsr1.h:684-769 (FSR_RCAS_DENOISE / PASSTHROUGH_ALPHA undefined: fsr_rcas.hlsl:1-4), reference order
template <bool U8>
__device__ __forceinline__ float3 rcas_filter(const float4 b, const float4 d, const float4 e, const float4 f,
                                              const float4 h, float sharp) {
  const float mn4R = fminf(fminf(b.x, fminf(d.x, f.x)), h.x), mx4R = fmaxf(fmaxf(b.x, fmaxf(d.x, f.x)), h.x);
  const float mn4G = fminf(fminf(b.y, fminf(d.y, f.y)), h.y), mx4G = fmaxf(fmaxf(b.y, fmaxf(d.y, f.y)), h.y);
  const float mn4B = fminf(fminf(b.z, fminf(d.z, f.z)), h.z), mx4B = fmaxf(fmaxf(b.z, fmaxf(d.z, f.z)), h.z);
  // limiters need full-precision reciprocals (:748-755)
  float lobe;
  if constexpr (U8) {
    // UNORM8 source: the limiter with its factors of 4 taken out, the same bits.  With mx, mn in {k/255} nothing here
    // is subnormal, so x4 and /4 are exact and commute with every rounding: fl(4mn-4) = 4 fl(mn-1) (fl(4mn) is exact),
    // 1/(4x) = (1/x)/4, so each hitMin / hitMax / lobe and the clamped max below are exactly 4x the reference's; the
    // x0.25 restores the reference's value BEFORE x sharp, so no assumption on `sharp` is needed.  Exhaustive host
    // check over every (mn, mx) code pair with mn <= mx: tests/test_rcas_limiter_host.py.
    const float hitMinR = mn4R * rcp_rn_unorm8_operand(mx4R);
    const float hitMinG = mn4G * rcp_rn_unorm8_operand(mx4G);
    const float hitMinB = mn4B * rcp_rn_unorm8_operand(mx4B);
    const float hitMaxR = (1.0f - mx4R) * rcp_rn_unorm8_operand(mn4R + (-1.0f));
    const float hitMaxG = (1.0f - mx4G) * rcp_rn_unorm8_operand(mn4G + (-1.0f));
    const float hitMaxB = (1.0f - mx4B) * rcp_rn_unorm8_operand(mn4B + (-1.0f));
    const float lobeR = fmaxf(-hitMinR, hitMaxR), lobeG = fmaxf(-hitMinG, hitMaxG), lobeB = fmaxf(-hitMinB, hitMaxB);
    lobe = fmaxf((float)(-4.0 * (0.25 - (1.0 / 16.0))), fminf(fmaxf(lobeR, fmaxf(lobeG, lobeB)), 0.0f)) * 0.25f * sharp;
  } else {
    const float hitMinR = mn4R * rcp_mode(4.0f * mx4R);
    const float hitMinG = mn4G * rcp_mode(4.0f * mx4G);
    const float hitMinB = mn4B * rcp_mode(4.0f * mx4B);
    const float hitMaxR = (1.0f - mx4R) * rcp_mode(4.0f * mn4R + (-4.0f));
    const float hitMaxG = (1.0f - mx4G) * rcp_mode(4.0f * mn4G + (-4.0f));
    const float hitMaxB = (1.0f - mx4B) * rcp_mode(4.0f * mn4B + (-4.0f));
    const float lobeR = fmaxf(-hitMinR, hitMaxR), lobeG = fmaxf(-hitMinG, hitMaxG), lobeB = fmaxf(-hitMinB, hitMaxB);
    lobe = fmaxf((float)(-(0.25 - (1.0 / 16.0))), fminf(fmaxf(lobeR, fmaxf(lobeG, lobeB)), 0.0f)) * sharp;
  }
  const float rcpL = prx_med_rcp(4.0f * lobe + 1.0f);
  return make_float3((lobe * b.x + lobe * d.x + lobe * h.x + lobe * f.x + e.x) * rcpL,
                     (lobe * b.y + lobe * d.y + lobe * h.y + lobe * f.y + e.y) * rcpL,
                     (lobe * b.z + lobe * d.z + lobe * h.z + lobe * f.z + e.z) * rcpL);
}

// fast math: (r,g) ride the FP32x2 pipe, b stays scalar; lobe*(b+d+h+f)+e regrouped
__device__ __forceinline__ float3 rcas_filter_fast(const float4 b, const float4 d, const float4 e, const float4 f,
                                                   const float4 h, float sharp) {
  const float mn4R = fminf(fminf(b.x, fminf(d.x, f.x)), h.x), mx4R = fmaxf(fmaxf(b.x, fmaxf(d.x, f.x)), h.x);
  const float mn4G = fminf(fminf(b.y, fminf(d.y, f.y)), h.y), mx4G = fmaxf(fmaxf(b.y, fmaxf(d.y, f.y)), h.y);
  const float mn4B = fminf(fminf(b.z, fminf(d.z, f.z)), h.z), mx4B = fmaxf(fmaxf(b.z, fmaxf(d.z, f.z)), h.z);
  const f2 mx = make_float2(mx4R, mx4G), mn = make_float2(mn4R, mn4G);
  const f2 dMin = mul2(mx, bc(4.0f)), dMax = fma2(mn, bc(4.0f), bc(-4.0f));
  const f2 hitMin = mul2(mn, make_float2(rcp_mode(dMin.x), rcp_mode(dMin.y)));
  const f2 hitMax = mul2(add2(bc(1.0f), make_float2(-mx4R, -mx4G)), make_float2(rcp_mode(dMax.x), rcp_mode(dMax.y)));
  const float hitMinB = mn4B * rcp_mode(4.0f * mx4B);
  const float hitMaxB = (1.0f - mx4B) * rcp_mode(fmaf(4.0f, mn4B, -4.0f));
  const float lobeR = fmaxf(-hitMin.x, hitMax.x), lobeG = fmaxf(-hitMin.y, hitMax.y), lobeB = fmaxf(-hitMinB, hitMaxB);
  const float lobe =
      fmaxf((float)(-(0.25 - (1.0 / 16.0))), fminf(fmaxf(lobeR, fmaxf(lobeG, lobeB)), 0.0f)) * sharp;
  const float rcpL = prx_med_rcp(fmaf(4.0f, lobe, 1.0f));
  const f2 sRG = add2(add2(make_float2(b.x, b.y), make_float2(d.x, d.y)), add2(make_float2(h.x, h.y), make_float2(f.x, f.y)));
  const float sB = (b.z + d.z) + (h.z + f.z);
  const f2 pRG = mul2(fma2(sRG, bc(lobe), make_float2(e.x, e.y)), bc(rcpL));
  return make_float3(pRG.x, pRG.y, fmaf(lobe, sB, e.z) * rcpL);
}

template <bool U8>
__device__ __forceinline__ float3 rcas_filter_mode(const float4 b, const float4 d, const float4 e, const float4 f,
                                                   const float4 h, float sharp) {
  if constexpr (kStrict) return rcas_filter<U8>(b, d, e, f, h, sharp);
  else return rcas_filter_fast(b, d, e, f, h, sharp);
}

// One-colour groups.  FsrRcasF reads the five texels b / d / e / f / h of a pixel's cross and nothing else (alpha
// included: it ignores it), so where every texel any cross of a group reads has the same RGB bits, every pixel of the
// group gets the same value, the filter of its first pixel.  Bit equality, not float equality: it holds for -0, NaN
// and HDR texels, in both math modes, with no lemma on the filter.  The union of the crosses is the group plus a
// 1-texel ring; this tests the whole 18 x 18 tile window w (corners included, which is conservative).  A partial group
// at the right / bottom image edge reads its ring from the zeros outside the image (Texture2D.Load), and every window
// texel past the edge is such a zero, so testing the whole window gives the answer the in-image part would.
// Called by all 32 lanes of a warp: two window rows per step (half-warps at columns 0-15 and 2-17), leaving at the
// first step that finds a second colour.
__device__ __forceinline__ bool rcas_flat_group(const float4 *__restrict__ w, int lane) {
  const float4 ref = w[kRcasTW + 1];
  const float4 *t = w + (lane & 15) + 2 * (lane >> 4);
  uint32_t diff = 0;
#pragma unroll 1
  for (int r = 0; diff == 0 && r < 18 * kRcasTW; r += 2 * kRcasTW) {
    const float4 u = t[r], v = t[r + kRcasTW];
    diff = __reduce_or_sync(0xFFFFFFFFu, (f2u(u.x) ^ f2u(ref.x)) | (f2u(u.y) ^ f2u(ref.y)) | (f2u(u.z) ^ f2u(ref.z)) |
                                             (f2u(v.x) ^ f2u(ref.x)) | (f2u(v.y) ^ f2u(ref.y)) | (f2u(v.z) ^ f2u(ref.z)));
  }
  return diff == 0;
}

// four adjacent output texels -> memory; one 128-bit store when the format is 4 bytes wide and alignment allows
template <int FOUT>
__device__ __forceinline__ void store_quad(const ImageRW &dst, bool vec, int x, int y, const float4 (&px)[4]) {
  uint8_t *row = dst.ptr + (size_t)y * dst.pitch;
  if constexpr (FOUT == OVRFSR_FORMAT_RGBA8 || FOUT == OVRFSR_FORMAT_RGB10A2) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if constexpr (FOUT == OVRFSR_FORMAT_RGBA8)
        w[i] = __byte_perm(__byte_perm(to_unorm8(px[i].x), to_unorm8(px[i].y), 0x0040), __byte_perm(to_unorm8(px[i].z), to_unorm8(px[i].w), 0x0040), 0x5410);
      else
        w[i] = to_unorm<1023>(px[i].x) | (to_unorm<1023>(px[i].y) << 10) | (to_unorm<1023>(px[i].z) << 20) | (to_unorm<3>(px[i].w) << 30);
    }
    if (vec && x + 3 < dst.w) {
      *reinterpret_cast<uint4 *>(row + (size_t)x * 4) = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (x + i < dst.w) reinterpret_cast<uint32_t *>(row)[x + i] = w[i];
    }
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (x + i < dst.w) store_texel<FOUT>(row, x + i, px[i].x, px[i].y, px[i].z, px[i].w);
  }
}

// One CTA: 64x32 output pixels; the (66 x 34) source box arrives by TMA (zero fill outside the image is exactly
// Texture2D.Load's behaviour) and is decoded once into a float4 tile.  One warp per 16x16 group; each lane walks a
// column of 8 rows and keeps the b / e / h texels of the cross in registers, so a pixel costs 3 shared loads, not 5.
// One tile per CTA on purpose: at 44 registers and 46 KB four CTAs share an SM and the hardware scheduler balances the
// 2808 tiles of a C2 eye.
// skipOutside (ctx path, EASU ran with EasuArgs::direct): outside-radius groups are already final in dst, so CTAs
// without an inside group return at once and outside groups of mixed tiles store nothing.
// PAIRED = skipOutside, OPQ = opaqueSrc as compile-time variants (the plain dispatch keeps its instruction stream).
// ANYIO = src (TMA == false only) and dst may be CUDA arrays (`io`); otherwise `io` is unused.
template <int FIN, int FOUT, bool TMA, bool PAIRED, bool OPQ, bool ANYIO>
__global__ void __launch_bounds__(kThreads, 2) rcas_kernel(const __grid_constant__ RcasArgs a,
                                                           const __grid_constant__ CUtensorMap srcMap,
                                                           const __grid_constant__ ArrayIO io) {
  __shared__ __align__(128) float4 sC[kRcasTH * kRcasTW];
  __shared__ __align__(128) uint32_t sRaw[TMA ? kRcasTH * kRcasRawW : 1];
  __shared__ uint64_t tileBar;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ox0 = blockIdx.x * kTileW, oy0 = blockIdx.y * kTileH;
  const int sx0 = ox0 - 1, sy0 = oy0 - 1;
  // same UNORM layout in and out: outside-radius texels pass through bit for bit
  constexpr bool kRawCopy = FIN == FOUT && (FIN == OVRFSR_FORMAT_RGBA8 || FIN == OVRFSR_FORMAT_RGB10A2);

  if constexpr (PAIRED) {
    // uniform per CTA: nothing of this tile is inside the radius -> nothing to do (and no TMA load is issued)
    bool any = false;
#pragma unroll
    for (int g = 0; g < 8; ++g)
      any = any || group_inside((blockIdx.x * 4u + (g & 3)) * 16u + 8u, (blockIdx.y * 2u + (g >> 2)) * 16u + 8u, a.centre, a.radiusSq);
    if (!any) return;
  }
  if constexpr (TMA) {
    if (tid == 0) {
      mbar_init(&tileBar, 1);
      fence_barrier_init();
      mbar_arrive_expect_tx(&tileBar, (uint32_t)(kRcasTH * kRcasRawW * 4));
      tma_load_2d(sRaw, &srcMap, ox0 - 4, sy0, &tileBar); // x origin 16-byte aligned: 3 unused texels on the left
    }
  }
  const uint32_t ggx = blockIdx.x * (kTileW / 16) + (warp & 3), ggy = blockIdx.y * (kTileH / 16) + (warp >> 2);
  const bool inside = group_inside(ggx * 16u + 8u, ggy * 16u + 8u, a.centre, a.radiusSq);

  if constexpr (TMA) {
    // a CTA whose 8 groups are all outside the radius and copy raw bytes needs no decoded tile at all
    const bool rawCopy = kRawCopy && a.tintGB == 1.0f;
    const int needTile = __syncthreads_or(inside || !rawCopy); // also orders the barrier init before the polls
    mbar_wait(&tileBar, 0);
    // the 34 x 66 texels as one flat index: 9 passes of the 256 threads, 97 % of the lanes busy (a row loop per warp with
    // a 32-wide column loop inside keeps 58 %: 66 columns take three column steps, 34 rows five row steps)
    if (needTile)
#pragma unroll
      for (int q = tid; q < kRcasTH * (kTileW + 2); q += kThreads) {
        const int ty = q / (kTileW + 2), tx = q - ty * (kTileW + 2);
        float4 c = decode_rgba<FIN>(sRaw[ty * kRcasRawW + tx + 3]);
        if constexpr (OPQ || PAIRED) c.w = 1.0f; // PAIRED: only the filter reads this tile, and it ignores alpha
        sC[ty * kRcasTW + tx] = c;
      }
  } else {
    // Texture2D.Load semantics: out of bounds reads 0 (fsr_rcas.hlsl:18)
#pragma unroll 3
    for (int q = tid; q < kRcasTH * (kTileW + 2); q += kThreads) {
      const int ty = q / (kTileW + 2), tx = q - ty * (kTileW + 2);
      const int gy = sy0 + ty, gx = sx0 + tx;
      float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gy >= 0 && gy < a.src.h && gx >= 0 && gx < a.src.w) {
        if constexpr (ANYIO && packed32(FIN)) {
          // a packed array decodes like the TMA landing zone of a pitched source would (decode_rgba: the math mode's
          // UNORM8 decode), so that the result does not depend on where the texels live
          c = io.src.on ? decode_rgba<FIN>(fetch_word_array<FIN>(io.src, gx, gy)) : fetch_texel<FIN>(a.src.ptr + (size_t)gy * a.src.pitch, gx);
        } else {
          c = get_texel<FIN, ANYIO>(a.src, io.src, gx, gy);
        }
        if constexpr (OPQ) c.w = 1.0f;
      }
      sC[ty * kRcasTW + tx] = c;
    }
  }
  __syncthreads();
  // inside groups whose crosses read one RGB store their first pixel's value (rcas_flat_group).  The skip is decided
  // here, per group, never at launch: which kernel a dispatch launches depends on formats and layouts only, not on
  // texel values (tests/test_gpu_float_signed.py relies on that for its coverage count).  Tested before the lanes
  // past the image edge leave, as the vote needs the whole warp, and by outside groups too: behind the radius test
  // ptxas keeps the store descriptor in vector registers and converts it before every store of the column.
  const bool flat = rcas_flat_group(sC + (warp >> 2) * 16 * kRcasTW + (warp & 3) * 16, lane) && inside;

  const int x = (int)ggx * 16 + (lane & 15);
  if (x >= a.dst.w) return;
  const int y0 = (int)ggy * 16 + (lane >> 4) * 8; // this lane's 8 consecutive rows
  const float4 *p = sC + (y0 - sy0) * kRcasTW + (x - sx0);
  if (inside) {
    float4 b = p[-kRcasTW], e = p[0];
    // pitched target: the store address advances by one row per pixel instead of being formed from (x, y)
    uint8_t *out = a.dst.ptr + (size_t)y0 * a.dst.pitch + (size_t)x * sizeof(texel_t<FOUT>);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int y = y0 + k;
      if (y >= a.dst.h) break;
      const float4 h = p[kRcasTW], d = p[-1], f = p[1];
      const float3 c = rcas_filter_mode<FIN == OVRFSR_FORMAT_RGBA8 || FIN == OVRFSR_FORMAT_BGRA8>(b, d, e, f, h, a.sharp);
      if constexpr (ANYIO) put_opaque<FOUT, ANYIO>(a.dst, io.dst, x, y, c.x, c.y, c.z);
      else *reinterpret_cast<texel_t<FOUT> *>(out) = encode_opaque<FOUT>(c.x, c.y, c.z);
      if (k == 0 && flat) {
        // the other rows of a one-colour group take row 0's value
        const int yEnd = min(y0 + 8, a.dst.h);
        if constexpr (ANYIO) {
          for (int yy = y0 + 1; yy < yEnd; ++yy) put_opaque<FOUT, ANYIO>(a.dst, io.dst, x, yy, c.x, c.y, c.z);
        } else {
          const texel_t<FOUT> v = encode_opaque<FOUT>(c.x, c.y, c.z);
#pragma unroll 1
          for (int yy = y0 + 1; yy < yEnd; ++yy) {
            out += a.dst.pitch;
            *reinterpret_cast<texel_t<FOUT> *>(out) = v;
          }
        }
        return;
      }
      b = e; e = h; p += kRcasTW; out += a.dst.pitch;
    }
  } else if constexpr (!PAIRED) {
    // OutputTexture[p] = mul * InputTexture[p], alpha included (fsr_rcas.hlsl:45-53)
    if constexpr (TMA && kRawCopy) {
      if (a.tintGB == 1.0f) {
        // debug tint off: mul == 1 and decode -> x1 -> encode is the identity on all 256 (1024, 4) codes (exhaustive
        // check in tests/test_host_logic.py), so the texel bits are copied straight from the TMA landing zone
        const uint32_t *q = sRaw + (y0 - sy0) * kRcasRawW + (x - sx0) + 3;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int y = y0 + k;
          if (y >= a.dst.h) break;
          put_word<FOUT, ANYIO>(a.dst, io.dst, x, y, q[k * kRcasRawW]);
        }
        return;
      }
    }
    for (int k = 0; k < 8; ++k) {
      const int y = y0 + k;
      if (y >= a.dst.h) break;
      const float4 e = p[k * kRcasTW];
      put_texel<FOUT, ANYIO>(a.dst, io.dst, x, y, 1.0f * e.x, a.tintGB * e.y, a.tintGB * e.z, 1.0f * e.w);
    }
  }
}

// Device self-test behind ovrfsr_selftest_rcp: every reciprocal operand strict RCAS can see with a UNORM8 source (mx
// and mn-1), fast sequence vs rcp.rn; for the operand +0 the sequence must give the NaN the filter relies on.
// out[0] = number of mismatching operands (must be 0), out[1] = operands checked.
__device__ __forceinline__ bool rcp_unorm8_operand_ok(float x) {
  const float r = rcp_rn_unorm8_operand(x);
  return x == 0.0f ? isnan(r) : f2u(r) == f2u(__frcp_rn(x));
}
__global__ void rcas_rcp_selftest_kernel(uint32_t *out) {
  const int k = threadIdx.x; // 0..255
  const float v = unorm8((float)k);
  int bad = 0;
  bad += !rcp_unorm8_operand_ok(v);
  bad += !rcp_unorm8_operand_ok(__fadd_rn(v, -1.0f));
  atomicAdd(&out[0], (uint32_t)bad);
  atomicAdd(&out[1], 2u);
}

} // inline namespace OVRFSR_MODE_NS
} // namespace ovrfsr

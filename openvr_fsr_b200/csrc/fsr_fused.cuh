// fsr_fused.cuh -- EASU -> (quantised intermediate) -> RCAS in ONE kernel for sm_90a.
//
// Replaces the two back-to-back dispatches of PostProcessor::ApplyPostProcess
// (src/postprocess/PostProcessor.cpp:586-594 in /root/reference: ApplyUpscaling then ApplySharpening) when both run
// on the FSR path.  The reference materialises the upscaled image in `upscaledTexture` (R8G8B8A8_UNORM, or
// R10G10B10A2_UNORM for a 10-bit source; DetermineOutputFormat, :63-74) and RCAS reads it back; here the intermediate
// of one 64x32 output tile plus the one-pixel ring RCAS needs around it lives in shared memory only:
//
//   1. the source box of the (66 x 34)-pixel region arrives by TMA (persistent CTAs, next tile's box in flight);
//      texels are decoded once, luma and the per-texel direction / length features follow (as in easu_kernel);
//   2. every pixel of the region gets its first-pass value -- FsrEasuF inside the radius, Bilinear() outside, by
//      the pixel's OWN 16x16 group, exactly what fsr_easu.hlsl:38-64 writes there -- which is then quantised to the
//      intermediate format and decoded again, bit for bit what the UAV store / Load pair of the two dispatches does
//      (pixels outside the image are zero: Texture2D.Load out of bounds, fsr_rcas.hlsl:18);
//   3. RCAS (or the outside-radius copy with the debug tint, fsr_rcas.hlsl:38-54) runs from that tile; a lane owns
//      four horizontally adjacent pixels and writes them with one 128-bit store.
//
// The ring is recomputed by the neighbouring tiles (+9.6 % first-pass work at 64x32); in exchange the intermediate
// is never written or read (C2: 79.7 -> 35.0 MB of algorithmic traffic per eye), its decode for RCAS disappears
// and the pass is one launch.  Tiles whose 6x4 groups are all outside the radius skip the feature / intermediate
// stages: bilinear, quantise, (tint,) store.  Results are bit-identical to easu_kernel followed by rcas_kernel in
// either math mode: the same device functions run on the same operands.
#pragma once

#include "fsr_kernels.cuh"

namespace ovrfsr {
inline namespace OVRFSR_MODE_NS {

constexpr int kFusedEW = kTileW + 2, kFusedEH = kTileH + 2; // first-pass region of one tile
constexpr int kFusedMS = 67;  // float4 row stride of the intermediate tile: 67 * 4 words = 12 (mod 32) keeps the
                              // eight rows a quarter-warp reads at once in distinct banks
constexpr int kFusedRing = 2 * kFusedEW + 2 * kTileH; // 196 ring pixels

struct FusedArgs {
  ImageRO src;
  ImageRW dst;
  float c0x, c0y, c0z, c0w;
  uint32_t centre[4];
  const uint32_t *centreDev; // nullptr: `centre`, `radiusSq`, `sharp`; else the ctx's latched block (load_centre, load_rcas_sharp)
  uint32_t radiusSq;
  float radW, radH;
  int tileW, tileH;   // shared source tile extent in texels (for the 66 x 34 region)
  float sharp;        // RCAS const0[0]
  float tintGB;       // 1 - debug*0.3
  int vecStore;       // dst base and pitch are 16-byte aligned: 128-bit stores allowed
  int finiteIn;       // float sources only: finite_in on every texel read (OVRFSR_FLAG_FINITE; the target is UNORM)
};

template <int FIN, int FMID, int FOUT, int TW, bool TMA>
__global__ void __launch_bounds__(kThreads, 2) fsr_fused_kernel(const __grid_constant__ FusedArgs a,
                                                                const __grid_constant__ CUtensorMap srcMap) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  __shared__ uint64_t tileBar;
  __shared__ BilinAxis sRowAxis[kFusedEH]; // Bilinear()'s row terms of the region (outside-radius pixels only)
  __shared__ BilinAxis sColAxis[kFusedEW]; // ... and its column terms
  __shared__ uint32_t sGroupMask;          // bit (gy * 6 + gx): group (tile group origin - 1 + g) is inside the radius
  const int th = a.tileH, tn = TW * th;
  float4 *sC = reinterpret_cast<float4 *>(smem_raw);  // decoded colour (r,g,b,1)
  float4 *sF = sC + tn;                               // (dirX, dirY, lenX, lenY) per texel
  float *sL = reinterpret_cast<float *>(sF + tn);     // luma*2 plane
  float4 *sM = reinterpret_cast<float4 *>(smem_raw + (((size_t)tn * 36 + 127) & ~(size_t)127)); // intermediate tile
  const int rawW = a.tileW + 4;                       // TMA box width (origin floored to 4 texels)
  uint32_t *sRaw = reinterpret_cast<uint32_t *>(reinterpret_cast<uint8_t *>(sM) + ((kFusedMS * kFusedEH * 16 + 127) & ~127));

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tilesX = (a.dst.w + kTileW - 1) / kTileW, tilesY = (a.dst.h + kTileH - 1) / kTileH;
  const int numTiles = tilesX * tilesY;
  constexpr bool kU8 = FMID == OVRFSR_FORMAT_RGBA8;

  auto tile_origin = [&](int t, int &ox0, int &oy0, int &sx0, int &sy0) {
    const int ty = t / tilesX, tx = t - ty * tilesX;
    ox0 = tx * kTileW; oy0 = ty * kTileH;
    // source tile origin: one texel left/above the 'f' texel of the region's first pixel (ox0 - 1, oy0 - 1)
    sx0 = (int)floorf(easu_pos(ox0 - 1, a.c0x, a.c0z)) - 1;
    sy0 = (int)floorf(easu_pos(oy0 - 1, a.c0y, a.c0w)) - 1;
  };

  int t = blockIdx.x;
  if constexpr (TMA) {
    if (tid == 0) {
      mbar_init(&tileBar, 1);
      fence_barrier_init();
      if (t < numTiles) {
        int ox0, oy0, sx0, sy0;
        tile_origin(t, ox0, oy0, sx0, sy0);
        mbar_arrive_expect_tx(&tileBar, (uint32_t)(rawW * th * 4));
        tma_load_2d(sRaw, &srcMap, sx0 & ~3, sy0, &tileBar); // box origin 16-byte aligned in x
      }
    }
    __syncthreads();
  }

  uint32_t centre[4], rsq[2];
  load_centre(centre, rsq, a.centre, a.radiusSq, a.centreDev);
  const float sharp = load_rcas_sharp(a.sharp, a.centreDev);
  uint32_t phase = 0;
  for (; t < numTiles; t += gridDim.x) {
    int ox0, oy0, sx0, sy0;
    tile_origin(t, ox0, oy0, sx0, sy0);
    const int ex0 = ox0 - 1, ey0 = oy0 - 1;
    const int tx0 = TMA ? (sx0 & ~3) : sx0;
    const int cols = TMA ? rawW : a.tileW;

    // radius test of the 6 x 4 groups the region touches (wrapping u32 like the shaders; groups left of / above the
    // image only hold out-of-image pixels, whose class is never used)
    if (warp == 0) {
      const uint32_t ggx = (uint32_t)(ox0 >> 4) - 1u + (uint32_t)(lane % 6), ggy = (uint32_t)(oy0 >> 4) - 1u + (uint32_t)(lane / 6);
      const bool in = lane < 24 && group_inside(ggx * 16u + 8u, ggy * 16u + 8u, centre, rsq[0], rsq[1]);
      const uint32_t m = __ballot_sync(0xffffffffu, in);
      if (lane == 0) sGroupMask = m;
    }

    // ---- stage 1: decode the clamped source tile once ----------------------------------------------------
    if constexpr (TMA) {
      mbar_wait(&tileBar, phase);
      phase ^= 1u;
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
              sL[ty * TW + tx] = c.z * 0.5f + (c.x * 0.5f + c.y); // luma*2, ffx_fsr1.h:363
              sC[ty * TW + tx] = c;
            }
          }
        }
      }
    } else {
      for (int ty = warp; ty < th; ty += kThreads / 32) {
        const int gy = clampi(sy0 + ty, 0, a.src.h - 1);
        const uint8_t *row = a.src.ptr + (size_t)gy * a.src.pitch;
        for (int tx = lane; tx < cols; tx += 32) {
          const int gx = clampi(tx0 + tx, 0, a.src.w - 1);
          float4 c = fetch_texel<FIN>(row, gx);
          if constexpr (!packed32(FIN)) {
            if (a.finiteIn) finite_in(c);
          }
          sL[ty * TW + tx] = c.z * 0.5f + (c.x * 0.5f + c.y);
          c.w = 1.0f;
          sC[ty * TW + tx] = c;
        }
      }
    }
    // Bilinear()'s separable terms for the region's rows and columns
    if (tid < kFusedEH) {
      const int y = ey0 + tid;
      if (y >= 0 && y < a.dst.h) sRowAxis[tid] = easu_bilinear_axis(y, a.radH, a.src.h, sy0, th);
    } else if (tid >= 64 && tid < 64 + kFusedEW) {
      const int x = ex0 + (tid - 64);
      if (x >= 0 && x < a.dst.w) sColAxis[tid - 64] = easu_bilinear_axis(x, a.radW, a.src.w, tx0, cols);
    }
    __syncthreads();
    const uint32_t gmask = sGroupMask;
    if constexpr (TMA) {
      // the landing zone is fully decoded: refill it with the NEXT tile's box while this tile is processed
      const int tn2 = t + gridDim.x;
      if (tid == 0 && tn2 < numTiles) {
        int nox, noy, nsx, nsy;
        tile_origin(tn2, nox, noy, nsx, nsy);
        fence_proxy_async();
        mbar_arrive_expect_tx(&tileBar, (uint32_t)(rawW * th * 4));
        tma_load_2d(sRaw, &srcMap, nsx & ~3, nsy, &tileBar);
      }
    }

    // this warp's 16x16 group (region group index (1 + (warp & 3), 1 + (warp >> 2)))
    const bool inside = (gmask >> ((1 + (warp >> 2)) * 6 + 1 + (warp & 3))) & 1u;

    if (gmask == 0u) {
      // ---- no group of the region is inside the radius: first pass = Bilinear(), second pass = copy (with tint).
      // lane -> 4 adjacent pixels of a row: r = lane & 7 (+8 on the second pass), chunk = lane >> 3
      const int gx0 = ox0 + (warp & 3) * 16 + (lane >> 3) * 4, lx = gx0 - ex0;
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const int y = oy0 + (warp >> 2) * 16 + (lane & 7) + 8 * p;
        if (y < a.dst.h && gx0 < a.dst.w) {
          const BilinAxis ay = sRowAxis[y - ey0];
          float4 px[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            px[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (gx0 + i < a.dst.w) { // columns beyond the image have no axis terms (and are not stored)
              const float3 c = easu_bilinear(sC, TW, sColAxis[lx + i], ay);
              if (FMID == FOUT && a.tintGB == 1.0f) {
                // store -> Load -> x1 -> store is the identity on UNORM codes: quantise once
                px[i] = make_float4(c.x, c.y, c.z, 1.0f);
              } else {
                const float4 m = mid_roundtrip<FMID>(c.x, c.y, c.z);
                px[i] = make_float4(1.0f * m.x, a.tintGB * m.y, a.tintGB * m.z, 1.0f * m.w);
              }
            }
          }
          store_quad<FOUT>(a.dst, a.vecStore != 0, gx0, y, px);
        }
      }
      __syncthreads(); // every warp is done with this tile before the next decode overwrites it
      continue;
    }

    // ---- stage 2: per-source-texel direction/length features -----------------------------------------------
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

    // ---- stage 3: first pass over the 66 x 34 region -> intermediate tile ------------------------------------
    // iterations 0..7: this warp's group, lane -> column, rows yFirst + 2k (as easu_kernel); iteration 8: one ring
    // pixel per thread (threads 0..195), classified by its own group
    {
      const int xc = ox0 + (warp & 3) * 16 + (lane & 15);
      const int yFirst = oy0 + (warp >> 2) * 16 + (lane >> 4);
      int xr, yr;
      if (tid < kFusedEW) { xr = ex0 + tid; yr = ey0; }
      else if (tid < 2 * kFusedEW) { xr = ex0 + tid - kFusedEW; yr = ey0 + kFusedEH - 1; }
      else if (tid < 2 * kFusedEW + kTileH) { xr = ex0; yr = oy0 + tid - 2 * kFusedEW; }
      else { xr = ex0 + kFusedEW - 1; yr = oy0 + tid - 2 * kFusedEW - kTileH; }
      const bool ringLane = tid < kFusedRing;
      const bool ringInside = (gmask >> (((yr - ey0 + 15) >> 4) * 6 + ((xr - ex0 + 15) >> 4))) & 1u;
#pragma unroll 1
      for (int k = 0; k < 9; ++k) {
        const bool ring = k == 8;
        if (ring && !ringLane) break;
        const int x = ring ? xr : xc, y = ring ? yr : yFirst + 2 * k;
        const bool in = ring ? ringInside : inside;
        float4 m = make_float4(0.f, 0.f, 0.f, 0.f); // outside the image: Texture2D.Load returns 0
        if (x >= 0 && x < a.dst.w && y >= 0 && y < a.dst.h) {
          float3 c;
          if (in) {
            const float ppx_full = easu_pos(x, a.c0x, a.c0z), ppy_full = easu_pos(y, a.c0y, a.c0w);
            const float fpx = floorf(ppx_full), fpy = floorf(ppy_full);
            const int o = ((int)fpy - sy0) * TW + (int)fpx - tx0;
            if constexpr (kStrict) c = easu_filter<TW>(sC + o, sF + o, ppx_full - fpx, ppy_full - fpy);
            else c = easu_filter_fast<TW>(sC + o, sF + o, ppx_full - fpx, ppy_full - fpy);
          } else {
            c = easu_bilinear(sC, TW, sColAxis[x - ex0], sRowAxis[y - ey0]);
          }
          m = mid_roundtrip<FMID>(c.x, c.y, c.z);
        }
        sM[(y - ey0) * kFusedMS + (x - ex0)] = m;
      }
    }
    __syncthreads();

    // ---- stage 4: RCAS (inside) / tinted copy (outside) from the intermediate tile; 4 adjacent pixels per lane ----
    {
      const int lx = 1 + (warp & 3) * 16 + (lane >> 3) * 4; // tile column of the lane's first pixel
      const int gx0 = ex0 + lx;
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const int ly = 1 + (warp >> 2) * 16 + (lane & 7) + 8 * p;
        const int y = ey0 + ly;
        if (y < a.dst.h && gx0 < a.dst.w) {
          const float4 *mid = sM + ly * kFusedMS + lx;
          float4 px[4];
          if (inside) {
            float4 mrow[6];
#pragma unroll
            for (int i = 0; i < 6; ++i) mrow[i] = mid[i - 1];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float3 c = rcas_filter_mode<kU8>(mid[i - kFusedMS], mrow[i], mrow[i + 1], mrow[i + 2], mid[i + kFusedMS], sharp);
              px[i] = make_float4(c.x, c.y, c.z, 1.0f);
            }
          } else {
            // OutputTexture[p] = mul * InputTexture[p] (fsr_rcas.hlsl:45-53); the intermediate's alpha is 1
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const float4 e = mid[i];
              px[i] = make_float4(1.0f * e.x, a.tintGB * e.y, a.tintGB * e.z, 1.0f * 1.0f);
            }
          }
          store_quad<FOUT>(a.dst, a.vecStore != 0, gx0, y, px);
        }
      }
    }
    __syncthreads(); // every warp is done with this tile before the next decode overwrites it
  }
}

} // inline namespace OVRFSR_MODE_NS
} // namespace ovrfsr

// nis_host.h -- CPU-side NISConfig setup (product code, header-only C++).
//
// What NVScalerUpdateConfig / NVSharpenUpdateConfig (src/nis/NIS_Config.h:144-255 in /root/reference)
// derive from the sharpness slider and the image sizes, with the argument pattern the mod uses
// (src/postprocess/PostProcessor.cpp:307-310,432-435): zero viewport origins, viewport == texture.
// Only the SDR branch exists here: the mod never passes an HDR mode.  Checked word-for-word against
// the reference header compiled as shipped in tests/test_host_logic.py.
#pragma once

#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstring>

#include "host_constants.h"

namespace ovrfsr {
namespace host {

// NISConfig, NIS_Config.h:37-77: 28 scalars, then the mod's uint4 centre + uint4 radius at byte 112
struct NisConfig {
  float kDetectRatio, kDetectThres, kMinContrastRatio, kRatioNorm;
  float kContrastBoost, kEps, kSharpStartY, kSharpScaleY;
  float kSharpStrengthMin, kSharpStrengthScale, kSharpLimitMin, kSharpLimitScale;
  float kScaleX, kScaleY, kDstNormX, kDstNormY;
  float kSrcNormX, kSrcNormY;
  uint32_t kInputViewportOriginX, kInputViewportOriginY, kInputViewportWidth, kInputViewportHeight;
  uint32_t kOutputViewportOriginX, kOutputViewportOriginY, kOutputViewportWidth, kOutputViewportHeight;
  float reserved0, reserved1;
  uint32_t imageCentre[4];
  uint32_t radius[4];
  uint32_t pad_[28];
};
static_assert(sizeof(NisConfig) == 256, "NISConfig is a 256-byte constant buffer");
static_assert(offsetof(NisConfig, imageCentre) == 112, "centre/radius sit at byte 112 (PostProcessor.cpp:310)");

// returns false (and leaves the tuning fields zero) when the scale is outside [0.5, 1], like the
// reference, whose caller ignores the result.
inline bool nis_update_config(NisConfig &c, float sharpness, uint32_t inW, uint32_t inH, uint32_t outW, uint32_t outH) {
  std::memset(&c, 0, sizeof(c));
  sharpness = std::max<float>(std::min<float>(1.f, sharpness), 0.f);
  const float slider = sharpness - 0.5f; // 0..1 -> -0.5..+0.5
  // two ranges: below 50% fades to no sharpening, above 50% is damped against over-sharpening
  const float minScale = slider >= 0.0f ? 1.25f : 1.0f;
  const float limitScale = slider >= 0.0f ? 1.25f : 1.0f;
  const float minContrast = 2.0f, maxContrast = 10.0f, startY = 0.45f, endY = 0.9f;
  const float strengthMin = std::max<float>(0.0f, 0.4f + slider * minScale * 1.2f);
  const float strengthMax = 1.6f + slider * 1.8f;
  const float limitMin = std::max<float>(0.1f, 0.14f + slider * limitScale * 0.32f);
  const float limitMax = 0.5f + slider * limitScale * 0.6f;

  c.kInputViewportWidth = inW; c.kInputViewportHeight = inH;
  c.kOutputViewportWidth = outW; c.kOutputViewportHeight = outH;
  if (inW == 0 || inH == 0 || outW == 0 || outH == 0) return false;
  c.kSrcNormX = 1.f / inW; c.kSrcNormY = 1.f / inH;
  c.kDstNormX = 1.f / outW; c.kDstNormY = 1.f / outH;
  c.kScaleX = inW / float(outW);
  c.kScaleY = inH / float(outH);
  if (c.kScaleX < 0.5f || c.kScaleX > 1.f || c.kScaleY < 0.5f || c.kScaleY > 1.f) return false;
  c.kDetectRatio = 1127.f / 1024.f;
  c.kDetectThres = 64.0f / 1024.0f;
  c.kMinContrastRatio = minContrast;
  c.kRatioNorm = 1.0f / (maxContrast - minContrast);
  c.kContrastBoost = 1.0f;
  c.kEps = 1.0f;
  c.kSharpStartY = startY;
  c.kSharpScaleY = 1.0f / (endY - startY);
  c.kSharpStrengthMin = strengthMin;
  c.kSharpStrengthScale = strengthMax - strengthMin;
  c.kSharpLimitMin = limitMin;
  c.kSharpLimitScale = limitMax - limitMin;
  return true;
}

inline bool make_nis_config(NisConfig &c, const ovrfsr_config &cfg, bool sharpenOnly, int eye, bool onlyOneEye,
                            uint32_t inW, uint32_t inH, uint32_t outW, uint32_t outH) {
  // NVSharpenUpdateConfig forwards the input size as the output size (NIS_Config.h:244-255); the mod
  // passes inputWidth/Height to it (PostProcessor.cpp:433), which equal the output size when renderScale == 1
  const bool ok = sharpenOnly ? nis_update_config(c, cfg.sharpness, inW, inH, inW, inH)
                              : nis_update_config(c, cfg.sharpness, inW, inH, outW, outH);
  c.reserved1 = cfg.debug_mode ? 1.f : 0.f;
  centre_radius(c.imageCentre, c.radius, cfg, eye, onlyOneEye, outW, outH);
  return ok;
}

// NVScaler's filter banks (NIS_Config.h:261-393), float[2][64 * 8]: coef_scale, then coef_usm, each 64 phases x
// kFilterSize (8) taps, 6 used.  Built on first use (nis_capi.cu).
const float *nis_coef_banks();

} // namespace host
} // namespace ovrfsr

// postprocessor.cpp -- see postprocessor.h.  Mirrors the control flow of
// /root/reference/src/postprocess/PostProcessor.cpp:123-194: guard, lazy init from the Config singleton,
// "log once, disable, pass through" on failure, handle/colour-space swap on success.
#include "postprocessor.h"

#include <cmath>
#include <cstdio>
#include <iostream>

Config &Config::Instance() {
  static Config instance;
  return instance;
}

static std::ostream *g_log = nullptr;
std::ostream &Log() { return g_log ? *g_log : std::clog; }
void SetLogStream(std::ostream *os) { g_log = os; }

namespace vr {

static ovrfsr_config config_from_singleton() {
  const Config &c = Config::Instance();
  ovrfsr_config k;
  ovrfsr_config_default(&k);
  k.fsr_enabled = c.fsrEnabled;
  k.use_nis = c.useNis;
  k.render_scale = c.renderScale;
  k.sharpness = c.sharpness;
  k.radius = c.radius;
  k.debug_mode = c.debugMode;
  for (int i = 0; i < 4; ++i) k.proj_centre[i] = c.projCentre[i];
  k.device = c.cudaDevice;
  k.math_mode = c.strictMath ? OVRFSR_MATH_STRICT : OVRFSR_MATH_FAST;
  k.flags = (c.fusedFsr ? OVRFSR_FLAG_FUSED_FSR : 0) | (c.srtm ? OVRFSR_FLAG_SRTM : 0) | (c.srtmNis ? OVRFSR_FLAG_SRTM_NIS : 0) |
            (c.finite ? OVRFSR_FLAG_FINITE : 0) | (c.perceptual ? OVRFSR_FLAG_PERCEPTUAL : 0);
  return k;
}

PostProcessor::~PostProcessor() {
  if (ctx) ovrfsr_destroy(ctx);
}

void PostProcessor::Apply(EVREye eEye, const Texture_t *pTexture, const VRTextureBounds_t *pBounds,
                          EVRSubmitFlags /*nSubmitFlags*/) {
  if (!enabled || pTexture == nullptr || pTexture->eType != TextureType_OvrFsrCuda || pTexture->handle == nullptr) {
    return;
  }
  static VRTextureBounds_t defaultBounds{0, 0, 1, 1};
  if (pBounds == nullptr) {
    pBounds = &defaultBounds;
  }
  if (!Config::Instance().fsrEnabled) {
    return;
  }
  const ovrfsr_image *texture = static_cast<const ovrfsr_image *>(pTexture->handle);

  if (!initialized) {
    // the reference re-reads the Config singleton whenever it (re)creates resources
    const ovrfsr_config k = config_from_singleton();
    int rc;
    {
      std::lock_guard<std::mutex> lock(ctxMutex); // SetFocus may create the ctx from another thread
      rc = ctx ? ovrfsr_set_config(ctx, &k) : ovrfsr_create(&ctx, &k);
    }
    if (rc != OVRFSR_OK) {
      Log() << "Resource creation failed, disabling (" << ovrfsr_status_string(rc) << ")\n";
      enabled = false;
      return;
    }
    // PostProcessor.cpp:504: Gamma, or Auto on a format OpenVR treats as sRGB (the _SRGB / _TYPELESS DXGI variants,
    // carried as tag bits of ovrfsr_image::format)
    inputIsSrgb = pTexture->eColorSpace == ColorSpace_Gamma ||
                  (pTexture->eColorSpace == ColorSpace_Auto && ovrfsr_format_considered_srgb(texture->format));
    Log() << "Creating post-processing resources\n";
    Log() << "Using " << (k.use_nis ? "NVIDIA Image Scaling" : "AMD FidelityFX SuperResolution") << "\n";
    initialized = true;
  }

  if (takeCapture) {
    takeCapture = false;
    ovrfsr_request_capture(ctx, captureDir);
  }
  const int onlyOneEye = std::abs(pBounds->uMax - pBounds->uMin) > .5f;
  const int eye = eEye == Eye_Right ? 1 : 0;
  ovrfsr_image out{};
  const ovrfsr_image *target = outputTargets[eye];
  const int rc = target ? ovrfsr_apply_into(ctx, eye, texture, onlyOneEye, target, stream)
                        : ovrfsr_apply(ctx, eye, texture, onlyOneEye, &out, stream);
  if (rc == OVRFSR_PASSTHROUGH) {
    return;
  }
  if (rc != OVRFSR_OK) {
    Log() << "Post-processing failed, disabling: " << ovrfsr_last_error(ctx) << "\n";
    enabled = false;
    return;
  }
  // the ctx's rule (PostProcessor.cpp:155-160): a shared texture is processed by the first Submit of a frame only
  const bool processed = onlyOneEye || submitCount == 0 || texture->data != lastSubmitted;
  lastSubmitted = texture->data;
  submitCount = (submitCount + 1) % 2;
  if (target) {
    // hand on the image that holds the result: this call's target, or the one the processing call wrote
    if (processed) lastTarget = target;
    const_cast<Texture_t *>(pTexture)->handle = const_cast<ovrfsr_image *>(lastTarget);
  } else {
    outputImage[eye] = out;
    const_cast<Texture_t *>(pTexture)->handle = &outputImage[eye];
  }
  // an sRGB-encoded output (OVRFSR_FLAG_PERCEPTUAL on a float eye into an 8-bit output) is gamma whatever the eye was.
  // The returned image says so with its tag; a caller's target has the ctx's output format, RGBA8 exactly when that is
  // 8-bit, and its tag is the caller's choice, so the ctx's config decides there.
  bool srgbOut = (out.format & OVRFSR_FORMAT_SRGB_BIT) != 0;
  if (target) {
    ovrfsr_config k{};
    const int layout = texture->format & OVRFSR_FORMAT_LAYOUT_MASK;
    const bool floatEye = layout == OVRFSR_FORMAT_RGBA16F || layout == OVRFSR_FORMAT_RGBA32F || layout == OVRFSR_FORMAT_RGB32F;
    srgbOut = ovrfsr_get_config(ctx, &k) == OVRFSR_OK && (k.flags & OVRFSR_FLAG_PERCEPTUAL) && floatEye &&
              (lastTarget->format & OVRFSR_FORMAT_LAYOUT_MASK) == OVRFSR_FORMAT_RGBA8;
  }
  const_cast<Texture_t *>(pTexture)->eColorSpace = inputIsSrgb || srgbOut ? ColorSpace_Gamma : ColorSpace_Auto;
}

void PostProcessor::Reset() {
  enabled = true;
  initialized = false;
  if (ctx) ovrfsr_reset(ctx);
  outputImage[0] = outputImage[1] = ovrfsr_image{};
  submitCount = 0;
  lastSubmitted = nullptr;
  lastTarget = nullptr;
}

void PostProcessor::TakeCapture(const char *directory) {
  std::snprintf(captureDir, sizeof(captureDir), "%s", directory ? directory : "");
  takeCapture = true;
}

bool PostProcessor::GetAverageGpuTimeMs(float *ms) { return ctx && ovrfsr_get_gpu_time_ms(ctx, ms) > 0; }

ovrfsr_ctx *PostProcessor::Context() {
  std::lock_guard<std::mutex> lock(ctxMutex);
  if (!ctx) {
    const ovrfsr_config k = config_from_singleton();
    if (ovrfsr_create(&ctx, &k) != OVRFSR_OK) ctx = nullptr;
  }
  return ctx;
}

// the focus lives in the ctx and survives the set_config of the first Apply and every Reset
bool PostProcessor::SetFocus(EVREye eEye, float x, float y) {
  ovrfsr_ctx *c = Context();
  return c && ovrfsr_set_focus(c, eEye == Eye_Right ? 1 : 0, x, y) == OVRFSR_OK;
}

bool PostProcessor::ClearFocus(EVREye eEye) {
  ovrfsr_ctx *c = Context();
  return c && ovrfsr_clear_focus(c, eEye == Eye_Right ? 1 : 0) == OVRFSR_OK;
}

// like the focus, the radius override lives in the ctx and survives the set_config of the first Apply and every Reset
bool PostProcessor::SetFocusRadius(EVREye eEye, float radius) {
  ovrfsr_ctx *c = Context();
  return c && ovrfsr_set_focus_radius(c, eEye == Eye_Right ? 1 : 0, radius) == OVRFSR_OK;
}

bool PostProcessor::ClearFocusRadius(EVREye eEye) {
  ovrfsr_ctx *c = Context();
  return c && ovrfsr_clear_focus_radius(c, eEye == Eye_Right ? 1 : 0) == OVRFSR_OK;
}

// the sharpness override lives in the ctx too: Reset and the set_config of the first Apply keep it
bool PostProcessor::SetSharpness(float sharpness) {
  ovrfsr_ctx *c = Context();
  return c && ovrfsr_set_sharpness(c, sharpness) == OVRFSR_OK;
}

bool PostProcessor::ClearSharpness() {
  ovrfsr_ctx *c = Context();
  return c && ovrfsr_clear_sharpness(c) == OVRFSR_OK;
}

} // namespace vr

// postprocessor.h -- C++ drop-in for vr::PostProcessor on the CUDA backend.
//
// Same public surface as /root/reference/src/postprocess/PostProcessor.h:12-13, so the Submit detours
// (src/postprocess/VrHooks.cpp:50-88) and ShutdownHooks (:155) compile against it unchanged:
//     postProcessor.Apply(eEye, pTexture, pBounds, nSubmitFlags);   postProcessor.Reset();
// Texture_t::handle carries an `ovrfsr_image*` (eType == TextureType_OvrFsrCuda) instead of an
// ID3D11Texture2D*.  All GPU work goes through the C ABI in include/ovrfsr.h.
#pragma once

#include <iosfwd>
#include <mutex>

#include "../../include/ovrfsr.h"
#include "config.h"
#include "openvr_min.h"

OVRFSR_API std::ostream &Log(); // Config.cpp:24-32 in the reference; here a settable stream (default std::clog)
OVRFSR_API void SetLogStream(std::ostream *os);

namespace vr {

class OVRFSR_API PostProcessor {
public:
  PostProcessor() = default;
  ~PostProcessor();
  PostProcessor(const PostProcessor &) = delete;
  PostProcessor &operator=(const PostProcessor &) = delete;

  void Apply(EVREye eEye, const Texture_t *pTexture, const VRTextureBounds_t *pBounds, EVRSubmitFlags nSubmitFlags);
  void Reset();

  // backend wiring the D3D11 version got from the texture itself (device/context, PostProcessor.cpp:500-501)
  void SetStream(void *cudaStream) { stream = cudaStream; }
  // mean GPU ms per frame in debugMode ("Average GPU processing time for upscale", PostProcessor.cpp:619-626)
  bool GetAverageGpuTimeMs(float *ms);
  // what the F7 hotkey does (`takeCapture = true`, PostProcessor.cpp:699-702): the next left-eye Apply writes its
  // output as capture_<time>_<fsr|nis>_s<..>_r<..>.dds into `directory` (the reference uses the DLL's directory)
  void TakeCapture(const char *directory);
  // Caller-owned output images (pitched or non-layered CUDA arrays, e.g. textures the compositor can read), one per
  // eye, outW x outH of the output format; nullptr / nullptr restores the ctx-owned outputs.  While set, Apply runs
  // ovrfsr_apply_into and hands on the image holding the result.  The pointers must stay valid while set.
  void SetOutputImages(const ovrfsr_image *left, const ovrfsr_image *right) {
    outputTargets[0] = left;
    outputTargets[1] = right;
  }
  // Foveation (ovrfsr_set_focus / ovrfsr_clear_focus): the radius mask of `eEye` centres on (x, y) in that eye's
  // normalised texture coordinates instead of its projection centre, from the next frame whose GPU work starts after
  // the call.  Callable from any thread (e.g. the eye tracker's), before the first Apply too.  false: rejected
  // (x / y not finite or outside [0, 1]).
  bool SetFocus(EVREye eEye, float x, float y);
  bool ClearFocus(EVREye eEye);
  // Dynamic foveation (ovrfsr_set_focus_radius / ovrfsr_clear_focus_radius): the radius mask of `eEye` uses `radius`
  // (the units of Config::radius) instead of Config::radius, from the next frame whose GPU work starts after the
  // call, with no Reset -- e.g. widened while the tracker's sample for that eye is invalid.  Same threading as
  // SetFocus.  false: rejected (radius not finite, negative or > 4).
  bool SetFocusRadius(EVREye eEye, float radius);
  bool ClearFocusRadius(EVREye eEye);
  // Live sharpness (ovrfsr_set_sharpness / ovrfsr_clear_sharpness): both eyes use `sharpness` instead of
  // Config::sharpness from the next frame whose GPU work starts after the call, with no Reset -- what the sharpness
  // hotkeys call after changing Config::sharpness.  Same threading as SetFocus.  false: rejected (not finite or
  // outside [0, 1]).
  bool SetSharpness(float sharpness);
  bool ClearSharpness();

private:
  ovrfsr_ctx *Context(); // creates the ctx on first use (no GPU work); guarded by ctxMutex
  std::mutex ctxMutex;
  bool enabled = true;
  bool initialized = false;
  bool inputIsSrgb = false;
  ovrfsr_ctx *ctx = nullptr;
  void *stream = nullptr;
  ovrfsr_image outputImage[2] = {};
  const ovrfsr_image *outputTargets[2] = {};
  // which Submit of a frame processes a shared texture (the ctx's eyeCount / lastSubmittedTexture), and the output
  // target that call wrote
  int submitCount = 0;
  const void *lastSubmitted = nullptr;
  const ovrfsr_image *lastTarget = nullptr;
  bool takeCapture = false;
  char captureDir[512] = {};
};

} // namespace vr

// pp_perceptual_selftest.cpp -- vr::PostProcessor with Config::perceptual on an RGBA16F stereo pair: the flag reaches
// the ctx through the drop-in, and the colour space handed on says what the RGBA8 output holds -- Gamma with the flag
// (sRGB-encoded), Auto without it (linear codes of a float eye, the reference's rule) -- with ctx-owned outputs and with
// SetOutputImages alike.  Each eye's output is written for the caller to compare with the checker.
// usage: pp_perceptual_selftest <in_left.rgba16f> <in_right.rgba16f> <w> <h> <renderScale> <sharpness> <radius>
//                               <perceptual 0|1> <use_targets 0|1> <out_left.rgba> <out_right.rgba>
// Built and run by tests/test_gpu_perceptual.py (nvcc, links the in-tree libovrfsr.so).
#include <cstdio>
#include <cstdlib>
#include <sstream>
#include <vector>

#include <cuda_runtime.h>

#include "postprocessor.h"

static int fail(const char *what) { std::fprintf(stderr, "pp_perceptual_selftest: %s\n", what); return 1; }

int main(int argc, char **argv) {
  if (argc != 12) return fail("bad arguments");
  const int w = std::atoi(argv[3]), h = std::atoi(argv[4]);
  const bool perceptual = std::atoi(argv[8]) != 0, useTargets = std::atoi(argv[9]) != 0;
  std::ostringstream log;
  SetLogStream(&log);
  Config &cfg = Config::Instance();
  cfg.fsrEnabled = true;
  cfg.renderScale = (float)std::atof(argv[5]);
  cfg.sharpness = (float)std::atof(argv[6]);
  cfg.radius = (float)std::atof(argv[7]);
  cfg.strictMath = true;
  cfg.perceptual = perceptual;
  const int outFmt = OVRFSR_FORMAT_RGBA8;
  const size_t outBpp = 4;

  ovrfsr_image eye[2], target[2];
  uint32_t ow = 0, oh = 0;
  ovrfsr_output_size(w, h, cfg.renderScale, &ow, &oh);
  for (int e = 0; e < 2; ++e) {
    std::vector<unsigned char> host((size_t)w * h * 8);
    FILE *f = std::fopen(argv[1 + e], "rb");
    if (!f || std::fread(host.data(), 1, host.size(), f) != host.size()) return fail("cannot read input");
    std::fclose(f);
    if (ovrfsr_image_alloc(&eye[e], w, h, OVRFSR_FORMAT_RGBA16F) != OVRFSR_OK) return fail("image alloc (no GPU?)");
    if (cudaMemcpy2D(eye[e].data, eye[e].pitch, host.data(), (size_t)w * 8, (size_t)w * 8, h, cudaMemcpyHostToDevice) != cudaSuccess)
      return fail("upload");
    if (useTargets && ovrfsr_image_alloc(&target[e], ow, oh, outFmt) != OVRFSR_OK) return fail("target alloc");
  }

  vr::PostProcessor postProcessor;
  if (useTargets) postProcessor.SetOutputImages(&target[0], &target[1]);
  vr::VRTextureBounds_t bounds{0.f, 0.f, 1.f, 1.f};
  for (int e = 0; e < 2; ++e) {
    vr::Texture_t t{&eye[e], vr::TextureType_OvrFsrCuda, vr::ColorSpace_Auto};
    void *origHandle = t.handle;
    postProcessor.Apply(e ? vr::Eye_Right : vr::Eye_Left, &t, &bounds, vr::Submit_Default);
    if (t.handle == origHandle) { std::fputs(log.str().c_str(), stderr); return fail("Apply did not swap the handle"); }
    const vr::EColorSpace want = perceptual ? vr::ColorSpace_Gamma : vr::ColorSpace_Auto;
    if (t.eColorSpace != want) return fail(perceptual ? "an sRGB output is not handed on as Gamma" : "a linear output is not handed on as Auto");
    const ovrfsr_image *out = static_cast<const ovrfsr_image *>(t.handle);
    const int wantTag = (perceptual && !useTargets) ? OVRFSR_FORMAT_SRGB_BIT : 0;
    if (out->format != (outFmt | wantTag)) return fail("the handed-on image has the wrong format tag");
    std::vector<unsigned char> res((size_t)out->width * out->height * outBpp);
    if (cudaMemcpy2D(res.data(), (size_t)out->width * outBpp, out->data, out->pitch, (size_t)out->width * outBpp, out->height,
                     cudaMemcpyDeviceToHost) != cudaSuccess)
      return fail("download");
    FILE *o = std::fopen(argv[10 + e], "wb");
    if (!o || std::fwrite(res.data(), 1, res.size(), o) != res.size()) return fail("cannot write output");
    std::fclose(o);
  }
  for (int e = 0; e < 2; ++e) {
    ovrfsr_image_free(&eye[e]);
    if (useTargets) ovrfsr_image_free(&target[e]);
  }
  std::printf("pp_perceptual_selftest: ok\n");
  return 0;
}

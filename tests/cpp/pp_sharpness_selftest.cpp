// pp_sharpness_selftest.cpp -- vr::PostProcessor::SetSharpness / ClearSharpness driven like the mod's sharpness hotkeys
// once they stop resetting: the sharpness is set before the first Apply (no ctx, no device work yet), survives a
// Reset, and ClearSharpness restores Config::sharpness.  Writes, per eye, the frame with the override and the frame
// after ClearSharpness.
// usage: pp_sharpness_selftest <in_left.rgba> <in_right.rgba> <w> <h> <renderScale> <sharpness> <radius> <useNis>
//                              <override> <set_left.rgba> <set_right.rgba> <clear_left.rgba> <clear_right.rgba>
// Built and run by tests/test_gpu_live_sharpness.py (nvcc, links the in-tree libovrfsr.so).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <sstream>
#include <vector>

#include <cuda_runtime.h>

#include "postprocessor.h"

static int fail(const char *what) { std::fprintf(stderr, "pp_sharpness_selftest: %s\n", what); return 1; }

int main(int argc, char **argv) {
  if (argc != 14) return fail("bad arguments");
  const int w = std::atoi(argv[3]), h = std::atoi(argv[4]);
  std::ostringstream log;
  SetLogStream(&log);
  Config &cfg = Config::Instance();
  cfg.fsrEnabled = true;
  cfg.renderScale = (float)std::atof(argv[5]);
  cfg.sharpness = (float)std::atof(argv[6]);
  cfg.radius = (float)std::atof(argv[7]);
  cfg.useNis = std::atoi(argv[8]) != 0;
  cfg.strictMath = true;
  const float sharpness = (float)std::atof(argv[9]);

  ovrfsr_image eye[2];
  for (int e = 0; e < 2; ++e) {
    std::vector<unsigned char> host((size_t)w * h * 4);
    FILE *f = std::fopen(argv[1 + e], "rb");
    if (!f || std::fread(host.data(), 1, host.size(), f) != host.size()) return fail("cannot read input");
    std::fclose(f);
    if (ovrfsr_image_alloc(&eye[e], w, h, OVRFSR_FORMAT_RGBA8) != OVRFSR_OK) return fail("image alloc (no GPU?)");
    if (cudaMemcpy2D(eye[e].data, eye[e].pitch, host.data(), (size_t)w * 4, (size_t)w * 4, h, cudaMemcpyHostToDevice) != cudaSuccess)
      return fail("upload");
  }

  vr::PostProcessor postProcessor;
  vr::VRTextureBounds_t bounds{0.f, 0.f, 1.f, 1.f};
  // before the first Apply: the drop-in creates its ctx, no GPU work happens
  if (!postProcessor.SetSharpness(sharpness)) return fail("SetSharpness rejected");
  // rejected values leave the sharpness alone
  if (postProcessor.SetSharpness(NAN) || postProcessor.SetSharpness(INFINITY) || postProcessor.SetSharpness(-0.01f) ||
      postProcessor.SetSharpness(1.01f))
    return fail("SetSharpness accepted an invalid sharpness");

  auto frame = [&](const char *outLeft, const char *outRight) -> int {
    for (int e = 0; e < 2; ++e) {
      vr::Texture_t t{&eye[e], vr::TextureType_OvrFsrCuda, vr::ColorSpace_Gamma};
      void *origHandle = t.handle;
      postProcessor.Apply(e ? vr::Eye_Right : vr::Eye_Left, &t, &bounds, vr::Submit_Default);
      if (t.handle == origHandle) { std::fputs(log.str().c_str(), stderr); return fail("Apply did not swap the handle"); }
      const ovrfsr_image *out = static_cast<const ovrfsr_image *>(t.handle);
      if (outLeft) {
        std::vector<unsigned char> res((size_t)out->width * out->height * 4);
        if (cudaMemcpy2D(res.data(), (size_t)out->width * 4, out->data, out->pitch, (size_t)out->width * 4, out->height,
                         cudaMemcpyDeviceToHost) != cudaSuccess)
          return fail("download");
        FILE *o = std::fopen(e ? outRight : outLeft, "wb");
        if (!o || std::fwrite(res.data(), 1, res.size(), o) != res.size()) return fail("cannot write output");
        std::fclose(o);
      }
    }
    return 0;
  };
  int rc = frame(nullptr, nullptr);
  if (rc) return rc;
  postProcessor.Reset(); // the override survives it
  if ((rc = frame(argv[10], argv[11])) != 0) return rc;
  if (!postProcessor.ClearSharpness()) return fail("ClearSharpness failed");
  if ((rc = frame(argv[12], argv[13])) != 0) return rc;
  for (int e = 0; e < 2; ++e) ovrfsr_image_free(&eye[e]);
  std::printf("pp_sharpness_selftest: ok\n");
  return 0;
}

// pp_focus_selftest.cpp -- vr::PostProcessor::SetFocus / ClearFocus driven like a gaze-tracking host would: the focus is
// set before the first Apply (no ctx, no device work yet), survives a Reset, and ClearFocus restores the projection
// centre.  Writes, per eye, the frame with the focus and the frame after ClearFocus.
// usage: pp_focus_selftest <in_left.rgba> <in_right.rgba> <w> <h> <renderScale> <sharpness> <radius> <useNis>
//                          <lx> <ly> <rx> <ry> <focus_left.rgba> <focus_right.rgba> <clear_left.rgba> <clear_right.rgba>
// Built and run by tests/test_gpu_focus.py (nvcc, links the in-tree libovrfsr.so).
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <sstream>
#include <vector>

#include <cuda_runtime.h>

#include "postprocessor.h"

static int fail(const char *what) { std::fprintf(stderr, "pp_focus_selftest: %s\n", what); return 1; }

int main(int argc, char **argv) {
  if (argc != 17) return fail("bad arguments");
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
  const float focus[2][2] = {{(float)std::atof(argv[9]), (float)std::atof(argv[10])}, {(float)std::atof(argv[11]), (float)std::atof(argv[12])}};

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
  // rejected arguments leave the focus alone
  if (postProcessor.SetFocus(vr::Eye_Left, NAN, 0.5f) || postProcessor.SetFocus(vr::Eye_Left, 0.5f, 1.5f))
    return fail("SetFocus accepted an invalid point");
  // before the first Apply: the drop-in creates its ctx, no GPU work happens
  for (int e = 0; e < 2; ++e)
    if (!postProcessor.SetFocus(e ? vr::Eye_Right : vr::Eye_Left, focus[e][0], focus[e][1])) return fail("SetFocus rejected");

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
  postProcessor.Reset(); // the focus survives it
  if ((rc = frame(argv[13], argv[14])) != 0) return rc;
  if (!postProcessor.ClearFocus(vr::Eye_Left) || !postProcessor.ClearFocus(vr::Eye_Right)) return fail("ClearFocus failed");
  if ((rc = frame(argv[15], argv[16])) != 0) return rc;
  for (int e = 0; e < 2; ++e) ovrfsr_image_free(&eye[e]);
  std::printf("pp_focus_selftest: ok\n");
  return 0;
}

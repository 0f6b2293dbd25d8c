// pp_finite_selftest.cpp -- vr::PostProcessor with Config::finite on an RGBA16F stereo pair holding +-inf and NaN
// texels: the flag reaches the ctx through the drop-in, and each eye's RGBA8 output is written for the caller to compare
// with the checker.
// usage: pp_finite_selftest <in_left.rgba16f> <in_right.rgba16f> <w> <h> <renderScale> <sharpness> <radius>
//                           <out_left.rgba> <out_right.rgba>
// Built and run by tests/test_gpu_finite.py (nvcc, links the in-tree libovrfsr.so).
#include <cstdio>
#include <cstdlib>
#include <sstream>
#include <vector>

#include <cuda_runtime.h>

#include "postprocessor.h"

static int fail(const char *what) { std::fprintf(stderr, "pp_finite_selftest: %s\n", what); return 1; }

int main(int argc, char **argv) {
  if (argc != 10) return fail("bad arguments");
  const int w = std::atoi(argv[3]), h = std::atoi(argv[4]);
  std::ostringstream log;
  SetLogStream(&log);
  Config &cfg = Config::Instance();
  cfg.fsrEnabled = true;
  cfg.renderScale = (float)std::atof(argv[5]);
  cfg.sharpness = (float)std::atof(argv[6]);
  cfg.radius = (float)std::atof(argv[7]);
  cfg.strictMath = true;
  cfg.finite = true;

  ovrfsr_image eye[2];
  for (int e = 0; e < 2; ++e) {
    std::vector<unsigned char> host((size_t)w * h * 8);
    FILE *f = std::fopen(argv[1 + e], "rb");
    if (!f || std::fread(host.data(), 1, host.size(), f) != host.size()) return fail("cannot read input");
    std::fclose(f);
    if (ovrfsr_image_alloc(&eye[e], w, h, OVRFSR_FORMAT_RGBA16F) != OVRFSR_OK) return fail("image alloc (no GPU?)");
    if (cudaMemcpy2D(eye[e].data, eye[e].pitch, host.data(), (size_t)w * 8, (size_t)w * 8, h, cudaMemcpyHostToDevice) != cudaSuccess)
      return fail("upload");
  }

  vr::PostProcessor postProcessor;
  vr::VRTextureBounds_t bounds{0.f, 0.f, 1.f, 1.f};
  for (int e = 0; e < 2; ++e) {
    vr::Texture_t t{&eye[e], vr::TextureType_OvrFsrCuda, vr::ColorSpace_Linear};
    void *origHandle = t.handle;
    postProcessor.Apply(e ? vr::Eye_Right : vr::Eye_Left, &t, &bounds, vr::Submit_Default);
    if (t.handle == origHandle) { std::fputs(log.str().c_str(), stderr); return fail("Apply did not swap the handle"); }
    const ovrfsr_image *out = static_cast<const ovrfsr_image *>(t.handle);
    if (out->format != OVRFSR_FORMAT_RGBA8) return fail("output is not RGBA8");
    std::vector<unsigned char> res((size_t)out->width * out->height * 4);
    if (cudaMemcpy2D(res.data(), (size_t)out->width * 4, out->data, out->pitch, (size_t)out->width * 4, out->height,
                     cudaMemcpyDeviceToHost) != cudaSuccess)
      return fail("download");
    FILE *o = std::fopen(argv[8 + e], "wb");
    if (!o || std::fwrite(res.data(), 1, res.size(), o) != res.size()) return fail("cannot write output");
    std::fclose(o);
  }
  for (int e = 0; e < 2; ++e) ovrfsr_image_free(&eye[e]);
  std::printf("pp_finite_selftest: ok\n");
  return 0;
}

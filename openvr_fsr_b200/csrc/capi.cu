// capi.cu -- implementation of include/ovrfsr.h: the state machine of vr::PostProcessor
// (src/postprocess/PostProcessor.cpp:123-194,498-638 in /root/reference) over CUDA resources,
// plus the stateless per-dispatch entry points.  No CPU fallback exists: if CUDA is unusable the
// calls fail with OVRFSR_ERR_CUDA.
#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <new>
#include <ctime>
#include <string>
#include <vector>

#include "array_io.h"
#include "host_constants.h"
#include "kernels.h"
#include "launch.cuh"
#include "nis_host.h"
#include "plan.h"

namespace ovrfsr {
static std::atomic<uint64_t> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
} // namespace ovrfsr

using namespace ovrfsr;

namespace {

constexpr int kQueryCount = 6; // QUERY_COUNT, PostProcessor.h:78

inline uint32_t bytes_per_pixel(int fmt) {
  return fmt == OVRFSR_FORMAT_RGBA32F ? 16u : (fmt == OVRFSR_FORMAT_RGB32F ? 12u : (fmt == OVRFSR_FORMAT_RGBA16F ? 8u : 4u));
}
inline bool valid_format(int fmt) { return fmt >= OVRFSR_FORMAT_RGBA8 && fmt <= OVRFSR_FORMAT_RGB32F; }
inline uint32_t align_up(uint32_t v, uint32_t a) { return (v + a - 1) / a * a; }

struct DeviceImage {
  Image img{};
  bool alloc(uint32_t w, uint32_t h, int fmt) {
    release();
    img.width = w; img.height = h; img.format = fmt; img.array_slices = 1; img.slice_pitch = 0;
    img.pitch = align_up(w * bytes_per_pixel(fmt), 256u);
    return cudaMalloc(&img.data, (size_t)img.pitch * h) == cudaSuccess;
  }
  // keep the image if it has this size and format, else reallocate it
  bool ensure(uint32_t w, uint32_t h, int fmt) {
    return (img.data && img.width == w && img.height == h && img.format == fmt) || alloc(w, h, fmt);
  }
  void release() {
    if (img.data) cudaFree(img.data);
    img = Image{};
  }
};

// linear device scratch for the host entry: PCIe copies are issued as ONE contiguous cudaMemcpyAsync each way
// (2-D pitched copies in opposite directions were measured not to overlap) and a
// small kernel moves rows between the tight host layout and the 256-byte-pitched device images.
struct DeviceBuffer {
  void *ptr = nullptr;
  size_t bytes = 0;
  bool ensure(size_t n) {
    if (n <= bytes) return true;
    release();
    if (cudaMalloc(&ptr, n) != cudaSuccess) { ptr = nullptr; return false; }
    bytes = n;
    return true;
  }
  void release() {
    if (ptr) cudaFree(ptr);
    ptr = nullptr; bytes = 0;
  }
};

// rows of `rowWords` 32-bit words from pitch `spitch` to pitch `dpitch` (bytes, multiples of 4); HBM-bound, ~10 us/eye
__global__ void __launch_bounds__(256) repitch_rows_kernel(uint8_t *__restrict__ dst, size_t dpitch, const uint8_t *__restrict__ src,
                                                           size_t spitch, uint32_t rowWords, uint32_t rows) {
  for (uint32_t y = blockIdx.y; y < rows; y += gridDim.y) {
    const uint32_t *s = reinterpret_cast<const uint32_t *>(src + (size_t)y * spitch);
    uint32_t *d = reinterpret_cast<uint32_t *>(dst + (size_t)y * dpitch);
    for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < rowWords; x += gridDim.x * blockDim.x) d[x] = s[x];
  }
}

cudaError_t repitch_rows(void *dst, size_t dpitch, const void *src, size_t spitch, size_t rowBytes, uint32_t rows, cudaStream_t s) {
  const uint32_t rowWords = (uint32_t)(rowBytes / 4);
  dim3 grid((rowWords + 1023) / 1024, rows < 4096 ? rows : 4096);
  return launch<repitch_rows_kernel>(grid, 256, 0, kNoOptIn, s, static_cast<uint8_t *>(dst), dpitch, static_cast<const uint8_t *>(src),
                                     spitch, rowWords, rows);
}

// R32G32B32_FLOAT -> RGBA32F, alpha 1 (a three-component view reads 1 in .w)
__global__ void __launch_bounds__(256) expand_rgb32f_kernel(float4 *__restrict__ dst, size_t dpitch, const float *__restrict__ src, size_t spitch,
                                                            uint32_t w, uint32_t h) {
  const uint32_t x = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y;
  if (x >= w || y >= h) return;
  const float *s = reinterpret_cast<const float *>(reinterpret_cast<const uint8_t *>(src) + (size_t)y * spitch) + 3 * (size_t)x;
  reinterpret_cast<float4 *>(reinterpret_cast<uint8_t *>(dst) + (size_t)y * dpitch)[x] = make_float4(s[0], s[1], s[2], 1.0f);
}
cudaError_t expand_rgb32f(const ovrfsr_image &src, const ovrfsr_image &dst, cudaStream_t s) {
  const dim3 grid((src.width + 255) / 256, src.height);
  return launch<expand_rgb32f_kernel>(grid, 256, 0, kNoOptIn, s, static_cast<float4 *>(dst.data), dst.pitch,
                                       static_cast<const float *>(src.data), src.pitch, src.width, src.height);
}

// The radius mask's focus and radius and the sharpness (ovrfsr_set_focus, ovrfsr_set_focus_radius,
// ovrfsr_set_sharpness).  `slot` (pinned host memory, one kLatchWords block per eye laid out as kernels.h describes) is
// what each apply's H2D copy reads when it runs on the GPU; it is written under `mu` only, each pair of words with one
// aligned 64-bit store, so a copy that overlaps an update sees whole pairs.  No CUDA call is made under `mu`.
struct Focus {
  std::mutex mu;
  bool set[2] = {false, false};
  float xy[2][2] = {};
  bool radiusSet[2] = {false, false};
  float radius[2] = {};     // in the units of ovrfsr_config::radius
  bool sharpSet = false;
  float sharpness = 0.f;    // in [0, 1]; one value for both eyes, like ovrfsr_config::sharpness
  // what the words are computed for: the ctx's config, layout, sizes and NIS pass at its last prepare_resources
  bool ready = false;
  ovrfsr_config cfg{};
  bool onlyOneEye = true;
  uint32_t inW = 0, inH = 0, outW = 0, outH = 0;
  bool nisSharpenOnly = false;
  uint32_t *slot = nullptr; // [2][kLatchWords], allocated by the first apply that needs it
  // some eye has a focus or a radius override, or the sharpness is overridden: applies copy the slot
  bool any() const { return set[0] || set[1] || radiusSet[0] || radiusSet[1] || sharpSet; }
};

} // namespace

struct ovrfsr_ctx {
  ovrfsr_config cfg{};
  // PostProcessor.h:16-24
  bool enabled = true;
  bool initialized = false;
  uint32_t inputWidth = 0, inputHeight = 0, outputWidth = 0, outputHeight = 0;
  bool textureContainsOnlyOneEye = true;
  int outFormat = OVRFSR_FORMAT_RGBA8;
  int inFormat = OVRFSR_FORMAT_RGBA8;
  // per-eye constant blocks (upscaleConstantsBuffer[2] / sharpenConstantsBuffer[2], PostProcessor.h:41,56)
  uint32_t upscaleConstants[2][24]{};
  uint32_t sharpenConstants[2][12]{};
  alignas(16) uint8_t nisScalerConfig[2][256]{};
  alignas(16) uint8_t nisSharpenConfig[2][256]{};
  Plan plan;
  // one set of intermediates/outputs PER EYE (the reference shares one; see ovrfsr.h): FSR's upscaled image, and the
  // image the last pass writes when the caller passes none
  DeviceImage upscaled[2], output[2];
  DeviceImage hostStage[2]; // device staging of host-submitted eyes (ovrfsr_apply_host)
  DeviceBuffer hostLinearIn[2], hostLinearOut[2];
  DeviceImage resolved[2];  // copiedTexture (PostProcessor.h:29): the resolved copy of a multisampled source
  DeviceImage expanded[2];  // RGBA32F copy of an R32G32B32_FLOAT source
  // F7 capture (takeCapture, PostProcessor.h:88 / PostProcessor.cpp:630-637)
  bool takeCapture = false;
  std::string captureDir, lastCapturePath;
  const void *lastSubmittedTexture = nullptr;
  Image lastOutput{};
  int eyeCount = 0;
  // debugMode profiling ring (PostProcessor.h:72-82)
  cudaEvent_t evStart[kQueryCount]{}, evEnd[kQueryCount]{};
  bool evPending[kQueryCount]{};
  bool evCreated = false;
  int currentQuery = 0;
  float summedGpuTime = 0.f;
  int countedQueries = 0;
  // ovrfsr_apply_pair: the right eye's chain runs on this stream between a fork and a join event
  cudaStream_t pairStream = nullptr;
  cudaEvent_t pairFork = nullptr, pairJoin = nullptr;
  // ovrfsr_set_focus / ovrfsr_set_focus_radius / ovrfsr_set_sharpness: `active` while some eye has a focus or a radius
  // override or the sharpness is overridden; then each apply copies its eye's slot block into `focusDev`
  // ([2][kLatchWords] words, device) at its head, and the kernels read their centre, radius and sharpness words from there
  Focus focus;
  std::atomic<bool> focusActive{false};
  uint32_t *focusDev = nullptr;
  std::string lastError;
};

namespace {

int fail(ovrfsr_ctx *ctx, int status, const char *what, cudaError_t e = cudaSuccess) {
  if (ctx) {
    ctx->lastError = what;
    if (e != cudaSuccess) { ctx->lastError += ": "; ctx->lastError += cudaGetErrorString(e); }
  }
  return status;
}

void release_resources(ovrfsr_ctx *c) {
  for (int e = 0; e < 2; ++e) { c->upscaled[e].release(); c->output[e].release(); c->hostStage[e].release(); c->hostLinearIn[e].release(); c->hostLinearOut[e].release(); c->resolved[e].release(); c->expanded[e].release(); }
  if (c->focusDev) { cudaFree(c->focusDev); c->focusDev = nullptr; }
  if (c->evCreated) {
    for (int i = 0; i < kQueryCount; ++i) { cudaEventDestroy(c->evStart[i]); cudaEventDestroy(c->evEnd[i]); c->evPending[i] = false; }
    c->evCreated = false;
  }
}

int select_device(ovrfsr_ctx *c) {
  if (c->cfg.device >= 0) {
    cudaError_t e = cudaSetDevice(c->cfg.device);
    if (e != cudaSuccess) return fail(c, OVRFSR_ERR_CUDA, "cudaSetDevice", e);
  }
  return OVRFSR_OK;
}

// the slot's words: host::centre_radius with each focused eye's proj_centre pair replaced by its focus, and radiusSq[k]
// the R^2 of the eye centre pair k is sourced from -- with that eye's radius override, if any, in place of cfg.radius.
// Block e of one-eye-per-texture submits takes both words from eye e; block 0 of a shared texture takes pair 0 from the
// left eye and pair 1 from the right (block 1 of a shared texture is never read).  The sharpness words of both blocks
// are those of the config with the override, if any, in place of cfg.sharpness, made by the very functions that
// prepare_resources builds the constant blocks with, so that they equal a configured ctx's bit for bit.
void write_focus_slot(Focus &f) {
  if (!f.slot || !f.ready) return;
  ovrfsr_config cfg = f.cfg;
  if (f.sharpSet) cfg.sharpness = f.sharpness;
  uint32_t rcas[12];
  host::make_sharpen_constants(rcas, cfg, 0, true, f.outW, f.outH);
  host::NisConfig nis;
  host::make_nis_config(nis, cfg, f.nisSharpenOnly, 0, true, f.inW, f.inH, f.outW, f.outH);
  const float nisSharp[4] = {nis.kSharpStrengthMin, nis.kSharpStrengthScale, nis.kSharpLimitMin, nis.kSharpLimitScale};
  for (int e = 0; e < 2; ++e)
    if (f.set[e]) { cfg.proj_centre[2 * e] = f.xy[e][0]; cfg.proj_centre[2 * e + 1] = f.xy[e][1]; }
  uint32_t eyeRsq[2];
  for (int e = 0; e < 2; ++e) {
    ovrfsr_config r = cfg;
    if (f.radiusSet[e]) r.radius = f.radius[e];
    uint32_t centre[4], radius[4];
    host::centre_radius(centre, radius, r, 0, true, f.outW, f.outH); // radius[1] does not depend on the eye or layout
    eyeRsq[e] = radius[1];
  }
  for (int b = 0; b < 2; ++b) {
    alignas(8) uint32_t words[kLatchNisSharp + 4] = {};
    uint32_t radius[4];
    host::centre_radius(words, radius, cfg, b, f.onlyOneEye, f.outW, f.outH);
    words[4] = eyeRsq[f.onlyOneEye ? b : 0];
    words[5] = eyeRsq[f.onlyOneEye ? b : 1];
    words[kLatchRcasSharp] = rcas[0];
    std::memcpy(words + kLatchNisSharp, nisSharp, sizeof(nisSharp));
    uint64_t pair[(kLatchNisSharp + 4) / 2];
    std::memcpy(pair, words, sizeof(pair));
    uint64_t *dst = reinterpret_cast<uint64_t *>(f.slot + kLatchWords * b);
    for (int k = 0; k < (kLatchNisSharp + 4) / 2; ++k) __atomic_store_n(&dst[k], pair[k], __ATOMIC_RELAXED);
  }
}

// head of an apply with a focus, a radius override or a sharpness override active: copy this eye's slot block to its
// device block on `s`, so the kernels of the apply see the words the slot holds when the copy runs (and a captured
// graph re-reads the slot on every replay)
int latch_focus(ovrfsr_ctx *c, int eye, cudaStream_t s, const uint32_t **centreDev) {
  Focus &f = c->focus;
  constexpr size_t kBytes = 2 * kLatchWords * sizeof(uint32_t);
  if (!f.slot) {
    uint32_t *slot = nullptr;
    cudaError_t e = cudaHostAlloc(reinterpret_cast<void **>(&slot), kBytes, cudaHostAllocPortable);
    if (e != cudaSuccess) return fail(c, OVRFSR_ERR_NOMEM, "allocating the focus slot", e);
    std::memset(slot, 0, kBytes); // the padding words
    std::lock_guard<std::mutex> lock(f.mu);
    f.slot = slot;
    write_focus_slot(f);
  }
  if (!c->focusDev) {
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&c->focusDev), kBytes);
    if (e != cudaSuccess) { c->focusDev = nullptr; return fail(c, OVRFSR_ERR_NOMEM, "allocating the focus block", e); }
  }
  cudaError_t e = cudaMemcpyAsync(c->focusDev + kLatchWords * eye, f.slot + kLatchWords * eye, kLatchWords * sizeof(uint32_t),
                                  cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) return fail(c, OVRFSR_ERR_CUDA, "focus copy", e);
  *centreDev = c->focusDev + kLatchWords * eye;
  return OVRFSR_OK;
}

// PostProcessor::PrepareResources, PostProcessor.cpp:498-561
int prepare_resources(ovrfsr_ctx *c, const ovrfsr_image *src) {
  c->inputWidth = src->width;
  c->inputHeight = src->height;
  c->inFormat = src->format;
  host::output_size(src->width, src->height, c->cfg.render_scale, &c->outputWidth, &c->outputHeight);
  if (c->outputWidth == 0 || c->outputHeight == 0) return fail(c, OVRFSR_ERR_INVALID, "output size is zero");
  // DetermineOutputFormat (PostProcessor.cpp:63-74): 10-bit sources keep a 10-bit target, everything else gets
  // RGBA8, unless the caller asks for a float output (extension)
  const bool tenBit = src->format == OVRFSR_FORMAT_RGB10A2;
  c->outFormat = c->cfg.output_format == OVRFSR_FORMAT_AUTO ? (tenBit ? OVRFSR_FORMAT_RGB10A2 : OVRFSR_FORMAT_RGBA8) : c->cfg.output_format;
  if (c->outFormat != OVRFSR_FORMAT_RGBA16F && c->outFormat != OVRFSR_FORMAT_RGBA32F &&
      c->outFormat != (tenBit ? OVRFSR_FORMAT_RGB10A2 : OVRFSR_FORMAT_RGBA8))
    return fail(c, OVRFSR_ERR_UNSUPPORTED, tenBit ? "output format for an RGB10A2 source must be RGB10A2, RGBA16F or RGBA32F"
                                                  : "output format must be RGBA8, RGBA16F or RGBA32F");
  c->plan = make_plan(c->cfg, src->format, c->outFormat);
  const Plan &p = c->plan;
  const bool one = c->textureContainsOnlyOneEye;
  const int neyes = one ? 2 : 1;
  for (int e = 0; e < neyes; ++e) {
    host::make_upscale_constants(c->upscaleConstants[e], c->cfg, e, one, c->inputWidth, c->inputHeight, c->outputWidth,
                                 c->outputHeight);
    host::make_sharpen_constants(c->sharpenConstants[e], c->cfg, e, one, c->outputWidth, c->outputHeight);
    ovrfsr_make_nis_config(c->nisScalerConfig[e], &c->cfg, 0, e, one, c->inputWidth, c->inputHeight, c->outputWidth,
                           c->outputHeight);
    ovrfsr_make_nis_config(c->nisSharpenConfig[e], &c->cfg, 1, e, one, c->inputWidth, c->inputHeight, c->outputWidth,
                           c->outputHeight);
    // the upscaled image only exists when EASU and RCAS run as two dispatches (the fused kernel keeps it in shared
    // memory; if a shape turns out not to be fusable it is allocated on first use)
    if (!p.nis && p.upscale && !p.tryFused && !c->upscaled[e].alloc(c->outputWidth, c->outputHeight, p.midFormat))
      return fail(c, OVRFSR_ERR_NOMEM, "allocating upscaled texture", cudaGetLastError());
    if (!c->output[e].alloc(c->outputWidth, c->outputHeight, c->outFormat))
      return fail(c, OVRFSR_ERR_NOMEM, p.nis && p.upscale ? "allocating upscaled texture" : "allocating sharpened texture",
                  cudaGetLastError());
  }
  if (c->cfg.debug_mode) {
    for (int i = 0; i < kQueryCount; ++i) {
      if (cudaEventCreate(&c->evStart[i]) != cudaSuccess || cudaEventCreate(&c->evEnd[i]) != cudaSuccess)
        return fail(c, OVRFSR_ERR_CUDA, "creating profiling events", cudaGetLastError());
      c->evPending[i] = false;
    }
    c->evCreated = true;
  }
  { // the slot words for the new config / layout / sizes (the focus and the overrides themselves survive resets)
    std::lock_guard<std::mutex> lock(c->focus.mu);
    Focus &f = c->focus;
    f.cfg = c->cfg; f.onlyOneEye = one; f.outW = c->outputWidth; f.outH = c->outputHeight; f.ready = true;
    f.inW = c->inputWidth; f.inH = c->inputHeight; f.nisSharpenOnly = !p.upscale; // the NISConfig the NIS pass takes
    write_focus_slot(f);
  }
  c->initialized = true;
  return OVRFSR_OK;
}

// harvest finished profiling samples (the GetData loop of PostProcessor.cpp:601-628, non-blocking)
void harvest_queries(ovrfsr_ctx *c) {
  if (!c->evCreated) return;
  for (int i = 0; i < kQueryCount; ++i) {
    if (!c->evPending[i] || cudaEventQuery(c->evEnd[i]) != cudaSuccess) continue;
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, c->evStart[i], c->evEnd[i]) == cudaSuccess) { c->summedGpuTime += ms; ++c->countedQueries; }
    c->evPending[i] = false;
  }
}

// PostProcessor::SaveTextureToFile, PostProcessor.cpp:640-657: staging copy, then the DDS writer (capture.cpp)
int save_capture(ovrfsr_ctx *c, const Image &img, cudaStream_t s) {
  ovrfsr_config named = c->cfg; // the name carries the sharpness override current when the capturing apply is issued
  {
    std::lock_guard<std::mutex> lock(c->focus.mu);
    if (c->focus.sharpSet) named.sharpness = c->focus.sharpness;
  }
  const size_t rowBytes = (size_t)img.width * bytes_per_pixel(img.format);
  std::vector<uint8_t> host(rowBytes * img.height);
  cudaError_t e = img.array ? cudaMemcpy2DFromArrayAsync(host.data(), rowBytes, static_cast<cudaArray_const_t>(img.data), 0, 0, rowBytes,
                                                         img.height, cudaMemcpyDeviceToHost, s)
                            : cudaMemcpy2DAsync(host.data(), rowBytes, img.data, img.pitch, rowBytes, img.height, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return fail(c, OVRFSR_ERR_CUDA, "capture read-back", e);
  char name[96];
  if (ovrfsr_capture_filename(&named, (int64_t)std::time(nullptr), name, sizeof(name)) != OVRFSR_OK)
    return fail(c, OVRFSR_ERR_INVALID, "capture file name");
  c->lastCapturePath = c->captureDir.empty() ? std::string(name) : c->captureDir + "/" + name;
  const ovrfsr_image h{host.data(), img.width, img.height, (uint32_t)rowBytes, img.format, 1, 0, 0};
  int rc = ovrfsr_dds_write(c->lastCapturePath.c_str(), &h);
  if (rc != OVRFSR_OK) { c->lastCapturePath.clear(); return fail(c, rc, "Error taking screen capture"); }
  return OVRFSR_OK;
}

// PostProcessor::ApplyPostProcess, PostProcessor.cpp:563-638 (the D3D11 binding save/restore and the Win32 hotkey
// polling stay in the caller; the F7 capture is served through ovrfsr_request_capture).  dst: the caller's image the
// last pass writes (ovrfsr_apply_into), else the ctx-owned output.
int apply_post_process(ovrfsr_ctx *c, int eye, const Image *src, Image *out, const Image *dst, cudaStream_t s) {
  const uint32_t *centreDev = nullptr;
  if (c->focusActive.load(std::memory_order_acquire)) {
    const int rc = latch_focus(c, eye, s, &centreDev);
    if (rc != OVRFSR_OK) return rc;
  }
  // GetInputView: array textures keep the right eye in slice 1 (PostProcessor.cpp:254-268)
  const int slice = (src->array_slices > 1 && eye == 1) ? 1 : 0;
  PassImage in = pass_image(*src, slice);
  cudaError_t e;
  if (src->sample_count > 1) { // GetInputView: multisampled sources are resolved into copiedTexture first (:219-226)
    DeviceImage &r = c->resolved[eye];
    if (!r.ensure(src->width, src->height, src->format))
      return fail(c, OVRFSR_ERR_NOMEM, "allocating the MSAA resolve target", cudaGetLastError());
    e = launch_resolve_msaa(in, (int)src->sample_count, pass_image(r.img), s);
    if (e != cudaSuccess) return fail(c, OVRFSR_ERR_CUDA, "MSAA resolve launch", e);
    in = pass_image(r.img);
  }
  if (src->format == OVRFSR_FORMAT_RGB32F) { // three-component float source: the kernels read it through an RGBA32F copy
    if (src->sample_count > 1) return fail(c, OVRFSR_ERR_UNSUPPORTED, "multisampled R32G32B32_FLOAT source");
    DeviceImage &x = c->expanded[eye];
    if (!x.ensure(src->width, src->height, OVRFSR_FORMAT_RGBA32F))
      return fail(c, OVRFSR_ERR_NOMEM, "allocating the RGBA32F copy of an RGB32F source", cudaGetLastError());
    ovrfsr_image sl = *src;
    sl.data = static_cast<uint8_t *>(src->data) + (size_t)slice * src->slice_pitch;
    e = expand_rgb32f(sl, x.img, s);
    if (e != cudaSuccess) return fail(c, OVRFSR_ERR_CUDA, "RGB32F expansion launch", e);
    in = pass_image(x.img);
  }
  int q = -1;
  if (c->evCreated) {
    harvest_queries(c);
    q = c->currentQuery;
    c->currentQuery = (c->currentQuery + 1) % kQueryCount;
    if (c->evPending[q]) q = -1; // oldest sample still in flight: skip this frame rather than block
    else cudaEventRecord(c->evStart[q], s);
  }
  // ApplyUpscaling and ApplySharpening (PostProcessor.cpp:586-594); the last pass writes fin
  const Plan &p = c->plan;
  const Image &fin = dst ? *dst : c->output[eye].img;
  const PassImage finPass = pass_image(fin);
  const Launchers &L = launchers(c->cfg.math_mode);
  bool fused = false;
  // the fused kernel has no array I/O: with an array source or destination the two dispatches run
  if (p.tryFused && !src->array && !fin.array) {
    // EASU and RCAS as one kernel; shapes it does not cover take the two dispatches below
    e = L.fsr_fused(in, finPass, c->upscaleConstants[eye], c->sharpenConstants[eye], s, centreDev, p.easuMaps);
    if (e == cudaSuccess) fused = true;
    else if (e != cudaErrorInvalidValue && e != cudaErrorInvalidConfiguration) return fail(c, OVRFSR_ERR_CUDA, "fused EASU+RCAS launch", e);
  }
  if (p.nis) {
    e = (p.upscale ? L.nis_scaler : L.nis_sharpen)(in, finPass, p.upscale ? c->nisScalerConfig[eye] : c->nisSharpenConfig[eye], s,
                                                    centreDev, p.nisMaps);
    if (e != cudaSuccess)
      return fail(c, (e == cudaErrorInvalidConfiguration || e == cudaErrorInvalidValue) ? OVRFSR_ERR_UNSUPPORTED : OVRFSR_ERR_CUDA,
                  p.upscale ? "NIS scaler dispatch" : "NIS sharpen dispatch", e);
  } else if (!fused) {
    if (p.upscale) { // paired: EASU writes its outside-radius groups to fin, and RCAS skips them
      DeviceImage &up = c->upscaled[eye];
      if (!up.ensure(c->outputWidth, c->outputHeight, p.midFormat))
        return fail(c, OVRFSR_ERR_NOMEM, "allocating upscaled texture", cudaGetLastError());
      const PassImage *direct = p.paired ? &finPass : nullptr;
      const float tint = 1.0f - (float)c->sharpenConstants[eye][3] * 0.3f;
      e = L.easu(in, pass_image(up.img), c->upscaleConstants[eye], s, direct, tint, centreDev, p.easuMaps);
      if (e != cudaSuccess) return fail(c, OVRFSR_ERR_CUDA, "EASU launch", e);
      in = pass_image(up.img);
    }
    e = L.rcas(in, finPass, c->sharpenConstants[eye], s, p.paired, centreDev, p.rcasMaps);
    if (e != cudaSuccess) return fail(c, OVRFSR_ERR_CUDA, "RCAS launch", e);
  }
  if (q >= 0) { cudaEventRecord(c->evEnd[q], s); c->evPending[q] = true; }
  *out = fin;
  if (c->takeCapture && eye == 0) { // PostProcessor.cpp:634-637
    c->takeCapture = false;
    int rc = save_capture(c, fin, s);
    if (rc != OVRFSR_OK) return rc;
  }
  return OVRFSR_OK;
}

// a pitched device or host image
int validate_image(const ovrfsr_image *im) {
  if (!im || !im->data || im->width == 0 || im->height == 0) return OVRFSR_ERR_INVALID;
  if (!valid_format(im->format)) return OVRFSR_ERR_UNSUPPORTED;
  const uint64_t rowEntries = (uint64_t)im->width * (im->sample_count > 1 ? im->sample_count : 1u);
  // rows and the base are aligned to the texel (to its 4-byte components for the 12-byte R32G32B32_FLOAT texel)
  const uint32_t align = im->format == OVRFSR_FORMAT_RGB32F ? 4u : bytes_per_pixel(im->format);
  if (im->sample_count > 32 || im->pitch < rowEntries * bytes_per_pixel(im->format) || (im->pitch % align) != 0) return OVRFSR_ERR_INVALID;
  if ((reinterpret_cast<uintptr_t>(im->data) % align) != 0) return OVRFSR_ERR_INVALID;
  return OVRFSR_OK;
}
// a pitched or array device image; dst: it is written by a kernel
int validate_image(const Image *im, bool dst = false) {
  if (im && im->array) return validate_array(*im, dst);
  return validate_image(static_cast<const ovrfsr_image *>(im));
}

// "Texture size changed, recreating resources" (PostProcessor.cpp:139-142); a format change does the same
void reset_if_source_changed(ovrfsr_ctx *c, const ovrfsr_image &src) {
  if (c->initialized && (src.width != c->inputWidth || src.height != c->inputHeight || src.format != c->inFormat)) ovrfsr_reset(c);
}

// ovrfsr_apply / ovrfsr_apply_into.  out: receives the output image (may be null); dst: the caller's output image (may
// be null)
int apply_impl(ovrfsr_ctx *ctx, int eye, const ovrfsr_image *src_tagged, int only_one_eye, ovrfsr_image *out,
               const ovrfsr_image *dst_tagged, void *stream) {
  if (!ctx || (eye != 0 && eye != 1)) return OVRFSR_ERR_INVALID;
  Image src_u{}, dst_u{};
  if (src_tagged) src_u = untagged(*src_tagged);
  if (dst_tagged) dst_u = untagged(*dst_tagged, false);
  // an sRGB-encoded output may be written into an RGBA8 destination tagged as sRGB (what ovrfsr_apply returns for it)
  if (src_tagged && dst_tagged && dst_u.format == (OVRFSR_FORMAT_RGBA8 | OVRFSR_FORMAT_SRGB_BIT) && srgb_output(ctx->cfg, src_u.format))
    dst_u.format = OVRFSR_FORMAT_RGBA8;
  const Image *src = src_tagged ? &src_u : nullptr, *dst = dst_tagged ? &dst_u : nullptr;
  // PostProcessor.cpp:124: disabled or unusable texture -> the frame passes through untouched
  if (!ctx->enabled || !ctx->cfg.fsr_enabled) return OVRFSR_PASSTHROUGH;
  int rc;
  // array images are inspected on the ctx's device
  if (((src && src->array) || (dst && dst->array)) && (rc = select_device(ctx)) != OVRFSR_OK) return rc;
  if ((rc = validate_image(src)) != OVRFSR_OK) return fail(ctx, rc, "invalid source image");
  if (dst && (rc = validate_image(dst, true)) != OVRFSR_OK) return fail(ctx, rc, "invalid destination image");
  if ((rc = select_device(ctx)) != OVRFSR_OK) return rc;
  reset_if_source_changed(ctx, *src);
  if (!ctx->initialized) {
    ctx->textureContainsOnlyOneEye = only_one_eye != 0; // PostProcessor.cpp:146
    rc = prepare_resources(ctx, src);
    if (rc != OVRFSR_OK) { // PostProcessor.cpp:148-152: "Resource creation failed, disabling"
      release_resources(ctx);
      ctx->enabled = false;
      return rc;
    }
  }
  if (dst && (dst->width != ctx->outputWidth || dst->height != ctx->outputHeight || dst->format != ctx->outFormat))
    return fail(ctx, OVRFSR_ERR_INVALID, "destination does not match the output size/format");
  // a single shared texture for both eyes is processed on the first Submit only (PostProcessor.cpp:155-160)
  if (ctx->eyeCount == 0 || ctx->textureContainsOnlyOneEye || src->data != ctx->lastSubmittedTexture) {
    rc = apply_post_process(ctx, ctx->textureContainsOnlyOneEye ? eye : 0, src, &ctx->lastOutput, dst,
                            static_cast<cudaStream_t>(stream));
    if (rc != OVRFSR_OK) return rc;
  }
  ctx->lastSubmittedTexture = src->data;
  ctx->eyeCount = (ctx->eyeCount + 1) % 2;
  if (out) {
    *out = tagged(ctx->lastOutput);
    if (ctx->plan.srgbOut) out->format |= OVRFSR_FORMAT_SRGB_BIT;
  }
  return OVRFSR_OK;
}

// ovrfsr_apply_pair / ovrfsr_apply_pair_into: the two apply_impl calls of one frame (out / dst as there, two each)
int apply_pair_impl(ovrfsr_ctx *ctx, const ovrfsr_image *src_left, const ovrfsr_image *src_right, int only_one_eye,
                    ovrfsr_image *out, const ovrfsr_image *dst, void *stream) {
  if (!ctx->enabled || !ctx->cfg.fsr_enabled) return OVRFSR_PASSTHROUGH;
  int rc = select_device(ctx);
  if (rc != OVRFSR_OK) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  ovrfsr_image *out0 = out ? &out[0] : nullptr, *out1 = out ? &out[1] : nullptr;
  const ovrfsr_image *dst0 = dst ? &dst[0] : nullptr, *dst1 = dst ? &dst[1] : nullptr;
  // one texture holding both eyes is processed once (PostProcessor.cpp:155-160): nothing to run side by side
  if (!only_one_eye) {
    if ((rc = apply_impl(ctx, 0, src_left, 0, out0, dst0, stream)) != OVRFSR_OK) return rc;
    return apply_impl(ctx, 1, src_right, 0, out1, dst1, stream);
  }
  if (!ctx->pairStream) {
    cudaError_t e = cudaStreamCreateWithFlags(&ctx->pairStream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->pairFork, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->pairJoin, cudaEventDisableTiming);
    if (e != cudaSuccess) return fail(ctx, OVRFSR_ERR_CUDA, "creating the pair stream", e);
  }
  // fork BEFORE the left eye is queued (the right eye must not wait for it), but queue the left eye first: it is the
  // call that (re)creates the resources when the source size changed
  cudaError_t e = cudaEventRecord(ctx->pairFork, s);
  if (e != cudaSuccess) return fail(ctx, OVRFSR_ERR_CUDA, "forking the pair stream", e);
  rc = apply_impl(ctx, 0, src_left, 1, out0, dst0, stream);
  if (rc != OVRFSR_OK) return rc;
  e = cudaStreamWaitEvent(ctx->pairStream, ctx->pairFork, 0);
  if (e != cudaSuccess) return fail(ctx, OVRFSR_ERR_CUDA, "forking the pair stream", e);
  rc = apply_impl(ctx, 1, src_right, 1, out1, dst1, ctx->pairStream);
  e = cudaEventRecord(ctx->pairJoin, ctx->pairStream);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(s, ctx->pairJoin, 0);
  if (e != cudaSuccess) return fail(ctx, OVRFSR_ERR_CUDA, "joining the pair stream", e);
  return rc;
}

} // namespace

extern "C" {

void ovrfsr_config_default(ovrfsr_config *cfg) {
  if (!cfg) return;
  std::memset(cfg, 0, sizeof(*cfg));
  cfg->struct_size = sizeof(ovrfsr_config);
  cfg->fsr_enabled = 0;   // Config.h:11
  cfg->use_nis = 0;       // Config.h:17
  cfg->render_scale = 1.f;
  cfg->sharpness = 0.75f;
  cfg->radius = 0.5f;
  cfg->debug_mode = 0;
  cfg->proj_centre[0] = cfg->proj_centre[1] = cfg->proj_centre[2] = cfg->proj_centre[3] = 0.5f;
  cfg->device = -1;
  cfg->output_format = OVRFSR_FORMAT_AUTO;
  cfg->math_mode = OVRFSR_MATH_STRICT; // parity first: bit-identical to the reference lines end to end
}

int ovrfsr_create(ovrfsr_ctx **out, const ovrfsr_config *cfg) {
  if (!out || !cfg || cfg->struct_size != sizeof(ovrfsr_config)) return OVRFSR_ERR_INVALID;
  if (!(cfg->render_scale > 0.f)) return OVRFSR_ERR_INVALID;
  ovrfsr_ctx *c = new (std::nothrow) ovrfsr_ctx();
  if (!c) return OVRFSR_ERR_NOMEM;
  c->cfg = *cfg;
  *out = c;
  return OVRFSR_OK;
}

void ovrfsr_destroy(ovrfsr_ctx *ctx) {
  if (ctx && ctx->pairStream) {
    cudaStreamSynchronize(ctx->pairStream);
    cudaEventDestroy(ctx->pairFork);
    cudaEventDestroy(ctx->pairJoin);
    cudaStreamDestroy(ctx->pairStream);
  }
  if (!ctx) return;
  if (ctx->initialized || ctx->hostStage[0].img.data || ctx->hostStage[1].img.data) {
    if (ctx->cfg.device >= 0) cudaSetDevice(ctx->cfg.device);
    release_resources(ctx);
  }
  if (ctx->focus.slot) cudaFreeHost(ctx->focus.slot);
  delete ctx;
}

int ovrfsr_reset(ovrfsr_ctx *ctx) {
  if (!ctx) return OVRFSR_ERR_INVALID;
  if (ctx->initialized) {
    if (ctx->cfg.device >= 0) cudaSetDevice(ctx->cfg.device);
    cudaDeviceSynchronize(); // outputs may still be in flight on the caller's stream
    release_resources(ctx);
  }
  ctx->enabled = true;
  ctx->initialized = false;
  ctx->lastSubmittedTexture = nullptr;
  ctx->lastOutput = Image{};
  ctx->eyeCount = 0;
  ctx->currentQuery = 0;
  ctx->summedGpuTime = 0.f;
  ctx->countedQueries = 0;
  return OVRFSR_OK;
}

int ovrfsr_set_config(ovrfsr_ctx *ctx, const ovrfsr_config *cfg) {
  if (!ctx || !cfg || cfg->struct_size != sizeof(ovrfsr_config) || !(cfg->render_scale > 0.f)) return OVRFSR_ERR_INVALID;
  int rc = ovrfsr_reset(ctx);
  ctx->cfg = *cfg;
  return rc;
}

int ovrfsr_set_focus(ovrfsr_ctx *ctx, int eye, float x, float y) {
  if (!ctx || (eye != 0 && eye != 1) || !(x >= 0.f && x <= 1.f) || !(y >= 0.f && y <= 1.f)) return OVRFSR_ERR_INVALID;
  Focus &f = ctx->focus;
  std::lock_guard<std::mutex> lock(f.mu);
  f.set[eye] = true;
  f.xy[eye][0] = x; f.xy[eye][1] = y;
  write_focus_slot(f);
  ctx->focusActive.store(true, std::memory_order_release);
  return OVRFSR_OK;
}

int ovrfsr_clear_focus(ovrfsr_ctx *ctx, int eye) {
  if (!ctx || (eye != 0 && eye != 1)) return OVRFSR_ERR_INVALID;
  Focus &f = ctx->focus;
  std::lock_guard<std::mutex> lock(f.mu);
  f.set[eye] = false;
  write_focus_slot(f); // graphs captured with a focus fall back to the projection centre
  ctx->focusActive.store(f.any(), std::memory_order_release);
  return OVRFSR_OK;
}

int ovrfsr_set_focus_radius(ovrfsr_ctx *ctx, int eye, float radius) {
  // 4 keeps R = 2 * outH, so R^2 <= 2^30 for outH <= 16384: the kernels' u32 square cannot wrap
  if (!ctx || (eye != 0 && eye != 1) || !(radius >= 0.f && radius <= 4.f)) return OVRFSR_ERR_INVALID;
  Focus &f = ctx->focus;
  std::lock_guard<std::mutex> lock(f.mu);
  f.radiusSet[eye] = true;
  f.radius[eye] = radius;
  write_focus_slot(f);
  ctx->focusActive.store(true, std::memory_order_release);
  return OVRFSR_OK;
}

int ovrfsr_clear_focus_radius(ovrfsr_ctx *ctx, int eye) {
  if (!ctx || (eye != 0 && eye != 1)) return OVRFSR_ERR_INVALID;
  Focus &f = ctx->focus;
  std::lock_guard<std::mutex> lock(f.mu);
  f.radiusSet[eye] = false;
  write_focus_slot(f); // graphs captured with an override fall back to ovrfsr_config::radius
  ctx->focusActive.store(f.any(), std::memory_order_release);
  return OVRFSR_OK;
}

int ovrfsr_set_sharpness(ovrfsr_ctx *ctx, float sharpness) {
  if (!ctx || !(sharpness >= 0.f && sharpness <= 1.f)) return OVRFSR_ERR_INVALID;
  Focus &f = ctx->focus;
  std::lock_guard<std::mutex> lock(f.mu);
  f.sharpSet = true;
  f.sharpness = sharpness;
  write_focus_slot(f);
  ctx->focusActive.store(true, std::memory_order_release);
  return OVRFSR_OK;
}

int ovrfsr_clear_sharpness(ovrfsr_ctx *ctx) {
  if (!ctx) return OVRFSR_ERR_INVALID;
  Focus &f = ctx->focus;
  std::lock_guard<std::mutex> lock(f.mu);
  f.sharpSet = false;
  write_focus_slot(f); // graphs captured with an override fall back to ovrfsr_config::sharpness
  ctx->focusActive.store(f.any(), std::memory_order_release);
  return OVRFSR_OK;
}

int ovrfsr_get_config(const ovrfsr_ctx *ctx, ovrfsr_config *cfg) {
  if (!ctx || !cfg) return OVRFSR_ERR_INVALID;
  *cfg = ctx->cfg;
  return OVRFSR_OK;
}

int ovrfsr_apply(ovrfsr_ctx *ctx, int eye, const ovrfsr_image *src, int only_one_eye, ovrfsr_image *out, void *stream) {
  if (!out) return OVRFSR_ERR_INVALID;
  return apply_impl(ctx, eye, src, only_one_eye, out, nullptr, stream);
}

int ovrfsr_apply_into(ovrfsr_ctx *ctx, int eye, const ovrfsr_image *src, int only_one_eye, const ovrfsr_image *dst, void *stream) {
  if (!dst) return OVRFSR_ERR_INVALID;
  return apply_impl(ctx, eye, src, only_one_eye, nullptr, dst, stream);
}

int ovrfsr_apply_pair(ovrfsr_ctx *ctx, const ovrfsr_image *src_left, const ovrfsr_image *src_right, int only_one_eye,
                      ovrfsr_image out[2], void *stream) {
  if (!ctx || !src_left || !src_right || !out) return OVRFSR_ERR_INVALID;
  return apply_pair_impl(ctx, src_left, src_right, only_one_eye, out, nullptr, stream);
}

int ovrfsr_apply_pair_into(ovrfsr_ctx *ctx, const ovrfsr_image *src_left, const ovrfsr_image *src_right, int only_one_eye,
                           const ovrfsr_image dst[2], void *stream) {
  if (!ctx || !src_left || !src_right || !dst) return OVRFSR_ERR_INVALID;
  return apply_pair_impl(ctx, src_left, src_right, only_one_eye, nullptr, dst, stream);
}

int ovrfsr_apply_host(ovrfsr_ctx *ctx, int eye, const ovrfsr_image *src_tagged, int only_one_eye,
                      const ovrfsr_image *dst_host, void *stream) {
  if (!ctx || (eye != 0 && eye != 1)) return OVRFSR_ERR_INVALID;
  Image src_untagged{};
  if (src_tagged) src_untagged = untagged(*src_tagged);
  const ovrfsr_image *src_host = src_tagged ? &src_untagged : nullptr;
  if (!ctx->enabled || !ctx->cfg.fsr_enabled) return OVRFSR_PASSTHROUGH;
  if (src_untagged.array) return fail(ctx, OVRFSR_ERR_UNSUPPORTED, "a host image cannot be a CUDA array");
  int rc = validate_image(src_host);
  if (rc != OVRFSR_OK) return fail(ctx, rc, "invalid host source image");
  if ((rc = validate_image(dst_host)) != OVRFSR_OK) return fail(ctx, rc, "invalid host destination image");
  if (src_host->sample_count > 1 || dst_host->sample_count > 1) return fail(ctx, OVRFSR_ERR_UNSUPPORTED, "multisampled host images");
  if ((rc = select_device(ctx)) != OVRFSR_OK) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // "Texture size changed, recreating resources" must happen BEFORE this eye is staged: the reset releases every
  // ctx-owned image, the staging images included
  reset_if_source_changed(ctx, *src_host);
  DeviceImage &st = ctx->hostStage[eye];
  if (!st.ensure(src_host->width, src_host->height, src_host->format))
    return fail(ctx, OVRFSR_ERR_NOMEM, "allocating host staging image", cudaGetLastError());
  const size_t rowBytes = (size_t)src_host->width * bytes_per_pixel(src_host->format);
  cudaError_t e;
  if (src_host->pitch == rowBytes) { // tight host rows: one contiguous PCIe copy, re-pitched on the device
    DeviceBuffer &lin = ctx->hostLinearIn[eye];
    if (!lin.ensure(rowBytes * src_host->height)) return fail(ctx, OVRFSR_ERR_NOMEM, "allocating linear upload buffer", cudaGetLastError());
    e = cudaMemcpyAsync(lin.ptr, src_host->data, rowBytes * src_host->height, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = repitch_rows(st.img.data, st.img.pitch, lin.ptr, rowBytes, rowBytes, src_host->height, s);
  } else {
    e = cudaMemcpy2DAsync(st.img.data, st.img.pitch, src_host->data, src_host->pitch, rowBytes, src_host->height,
                          cudaMemcpyHostToDevice, s);
  }
  if (e != cudaSuccess) return fail(ctx, OVRFSR_ERR_CUDA, "host->device copy", e);
  ovrfsr_image out{};
  rc = ovrfsr_apply(ctx, eye, &st.img, only_one_eye, &out, stream);
  if (rc != OVRFSR_OK) return rc;
  if (dst_host->width != out.width || dst_host->height != out.height || dst_host->format != (out.format & ~OVRFSR_FORMAT_SRGB_BIT))
    return fail(ctx, OVRFSR_ERR_INVALID, "host destination does not match the output size/format");
  const size_t outRowBytes = (size_t)out.width * bytes_per_pixel(out.format);
  if (dst_host->pitch == outRowBytes && out.pitch != outRowBytes) {
    DeviceBuffer &lin = ctx->hostLinearOut[eye];
    if (!lin.ensure(outRowBytes * out.height)) return fail(ctx, OVRFSR_ERR_NOMEM, "allocating linear download buffer", cudaGetLastError());
    e = repitch_rows(lin.ptr, outRowBytes, out.data, out.pitch, outRowBytes, out.height, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(dst_host->data, lin.ptr, outRowBytes * out.height, cudaMemcpyDeviceToHost, s);
  } else {
    e = cudaMemcpy2DAsync(dst_host->data, dst_host->pitch, out.data, out.pitch, outRowBytes, out.height, cudaMemcpyDeviceToHost, s);
  }
  return e == cudaSuccess ? OVRFSR_OK : fail(ctx, OVRFSR_ERR_CUDA, "device->host copy", e);
}

int ovrfsr_request_capture(ovrfsr_ctx *ctx, const char *directory) {
  if (!ctx) return OVRFSR_ERR_INVALID;
  ctx->captureDir = directory ? directory : "";
  ctx->takeCapture = true; // the hotkey sets the flag, the next left-eye frame is saved (PostProcessor.cpp:699-702,634)
  return OVRFSR_OK;
}

const char *ovrfsr_last_capture_path(const ovrfsr_ctx *ctx) { return ctx ? ctx->lastCapturePath.c_str() : ""; }

int ovrfsr_resolve_msaa(const ovrfsr_image *src, const ovrfsr_image *dst, void *stream) {
  Image src_untagged_{};
  if (src) { src_untagged_ = untagged(*src); src = &src_untagged_; }
  if (src_untagged_.array || (dst && untagged(*dst).array)) return OVRFSR_ERR_UNSUPPORTED; /* no array I/O */
  int rc = validate_image(src);
  if (rc != OVRFSR_OK || (rc = validate_image(dst)) != OVRFSR_OK) return rc;
  if (src->sample_count < 2 || dst->sample_count > 1 || src->format != dst->format || src->width != dst->width || src->height != dst->height)
    return OVRFSR_ERR_INVALID;
  cudaError_t e = launch_resolve_msaa(pass_image(src_untagged_), (int)src->sample_count, pass_image(untagged(*dst, false)), static_cast<cudaStream_t>(stream));
  return e == cudaSuccess ? OVRFSR_OK : (e == cudaErrorInvalidValue ? OVRFSR_ERR_UNSUPPORTED : OVRFSR_ERR_CUDA);
}

int ovrfsr_expand_rgb32f(const ovrfsr_image *src, const ovrfsr_image *dst, void *stream) {
  Image src_untagged_{};
  if (src) { src_untagged_ = untagged(*src); src = &src_untagged_; }
  if (src_untagged_.array || (dst && untagged(*dst).array)) return OVRFSR_ERR_UNSUPPORTED; /* no array I/O */
  int rc = validate_image(src);
  if (rc != OVRFSR_OK || (rc = validate_image(dst)) != OVRFSR_OK) return rc;
  if (src->format != OVRFSR_FORMAT_RGB32F || dst->format != OVRFSR_FORMAT_RGBA32F || src->width != dst->width || src->height != dst->height ||
      src->sample_count > 1 || dst->sample_count > 1)
    return OVRFSR_ERR_INVALID;
  return expand_rgb32f(*src, *dst, static_cast<cudaStream_t>(stream)) == cudaSuccess ? OVRFSR_OK : OVRFSR_ERR_CUDA;
}

int ovrfsr_format_considered_srgb(int32_t f) {
  if (f < 0) return 0;
  const int layout = f & OVRFSR_FORMAT_LAYOUT_MASK;
  const bool eightBit = layout == OVRFSR_FORMAT_RGBA8 || layout == OVRFSR_FORMAT_BGRA8 || layout == OVRFSR_FORMAT_BGRX8;
  if ((f & OVRFSR_FORMAT_SRGB_BIT) && eightBit) return 1;                                            // PostProcessor.cpp:78-81
  if ((f & OVRFSR_FORMAT_TYPELESS_BIT) && (eightBit || layout == OVRFSR_FORMAT_RGB10A2)) return 1;  // :82-87
  return 0;
}

// ---- stateless dispatches (ApplyUpscaling / ApplySharpening, PostProcessor.cpp:385-401,483-496) --------------
static int check_pair(const Image *src, const Image *dst) {
  int rc = validate_image(src);
  if (rc != OVRFSR_OK) return rc;
  if ((rc = validate_image(dst, true)) != OVRFSR_OK) return rc;
  if (src->format == OVRFSR_FORMAT_RGB32F) return OVRFSR_ERR_UNSUPPORTED;                                   /* expand first (ovrfsr_expand_rgb32f / ovrfsr_apply) */
  if (dst->format == OVRFSR_FORMAT_BGRX8 || dst->format == OVRFSR_FORMAT_RGB32F) return OVRFSR_ERR_UNSUPPORTED; /* source-only formats */
  if (src->sample_count > 1 || dst->sample_count > 1) return OVRFSR_ERR_UNSUPPORTED; /* resolve first (ovrfsr_resolve_msaa / ovrfsr_apply) */
  if (dst->format == OVRFSR_FORMAT_BGRA8) return OVRFSR_ERR_UNSUPPORTED; /* outputs are RGBA8 / RGB10A2 (reference) or float */
  if ((dst->format == OVRFSR_FORMAT_RGB10A2) != (src->format == OVRFSR_FORMAT_RGB10A2) && dst->format != OVRFSR_FORMAT_RGBA16F &&
      dst->format != OVRFSR_FORMAT_RGBA32F)
    return OVRFSR_ERR_UNSUPPORTED; /* UNORM targets follow DetermineOutputFormat: 10-bit in <-> 10-bit out */
  return OVRFSR_OK;
}

// one image of a stateless NIS dispatch (dst: it is written).  Unlike check_pair, it refuses a format or multisampling
// before it looks at the pitch.
static int check_nis_image(const Image *im, bool isDst) {
  if (!im || !im->data || im->width == 0 || im->height == 0) return OVRFSR_ERR_INVALID;
  if (im->format < OVRFSR_FORMAT_RGBA8 || im->format > OVRFSR_FORMAT_BGRX8) return OVRFSR_ERR_UNSUPPORTED; /* RGB32F: expand first */
  if ((isDst && (im->format == OVRFSR_FORMAT_BGRA8 || im->format == OVRFSR_FORMAT_BGRX8)) || im->sample_count > 1) return OVRFSR_ERR_UNSUPPORTED;
  if (im->array) return validate_array(*im, isDst);
  const uint32_t bpp = bytes_per_pixel(im->format);
  if (im->pitch < im->width * bpp || im->pitch % bpp || reinterpret_cast<uintptr_t>(im->data) % bpp) return OVRFSR_ERR_INVALID;
  return OVRFSR_OK;
}

// the pass flags of a stateless dispatch: OVRFSR_OK, or the status to return (checked after the images)
static int check_pass_flags(const Image *src, int pass_flags) {
  if (pass_flags & ~(kMapsIn | kMapsOut)) return OVRFSR_ERR_INVALID;
  if (pass_flags && src->format != OVRFSR_FORMAT_RGBA16F && src->format != OVRFSR_FORMAT_RGBA32F) return OVRFSR_ERR_UNSUPPORTED;
  return OVRFSR_OK;
}

// the status of a stateless dispatch's launch.  cudaErrorInvalidValue is a shape or format the pass does not cover; so
// is cudaErrorInvalidConfiguration where `configUnsupported` (EASU, fused and NIS refuse a scale with it).  RCAS and
// CAS refuse nothing with it, so there it is a failed launch.
static int launch_status(cudaError_t e, bool configUnsupported) {
  if (e == cudaErrorInvalidValue || (configUnsupported && e == cudaErrorInvalidConfiguration)) return OVRFSR_ERR_UNSUPPORTED;
  return e == cudaSuccess ? OVRFSR_OK : OVRFSR_ERR_CUDA;
}

// the two images of a stateless dispatch, untagged; null where the caller passed null
struct DispatchPair {
  Image s{}, d{};
  const Image *src = nullptr, *dst = nullptr;
  DispatchPair(const ovrfsr_image *src_tagged, const ovrfsr_image *dst_tagged) {
    if (src_tagged) { s = untagged(*src_tagged); src = &s; }
    if (dst_tagged) { d = untagged(*dst_tagged, false); dst = &d; }
  }
  bool any_array() const { return (src && src->array) || (dst && dst->array); }
};

int ovrfsr_dispatch_fsr_easu(const ovrfsr_image *src_tagged, const ovrfsr_image *dst_tagged, const uint32_t consts[24], int math_mode,
                             void *stream) {
  return ovrfsr_dispatch_fsr_easu_ex(src_tagged, dst_tagged, consts, math_mode, 0, stream);
}

int ovrfsr_dispatch_fsr_easu_ex(const ovrfsr_image *src_tagged, const ovrfsr_image *dst_tagged, const uint32_t consts[24], int math_mode,
                                int pass_flags, void *stream) {
  const DispatchPair io(src_tagged, dst_tagged);
  const Image *src = io.src, *dst = io.dst;
  if (!consts) return OVRFSR_ERR_INVALID;
  int rc = check_pair(src, dst);
  if (rc != OVRFSR_OK || (rc = check_pass_flags(src, pass_flags)) != OVRFSR_OK) return rc;
  return launch_status(launchers(math_mode).easu(pass_image(*src), pass_image(*dst), consts, static_cast<cudaStream_t>(stream), nullptr,
                                                 1.0f, nullptr, pass_flags),
                       /*configUnsupported=*/true);
}

int ovrfsr_dispatch_fsr_fused(const ovrfsr_image *src_tagged, const ovrfsr_image *dst_tagged, const uint32_t upscale_consts[24],
                              const uint32_t sharpen_consts[12], int math_mode, void *stream) {
  const DispatchPair io(src_tagged, dst_tagged);
  const Image *src = io.src, *dst = io.dst;
  if (!upscale_consts || !sharpen_consts) return OVRFSR_ERR_INVALID;
  if (io.any_array()) return OVRFSR_ERR_UNSUPPORTED; /* the fused kernel has no array I/O */
  int rc = check_pair(src, dst);
  if (rc != OVRFSR_OK) return rc;
  return launch_status(launchers(math_mode).fsr_fused(pass_image(*src), pass_image(*dst), upscale_consts, sharpen_consts,
                                                      static_cast<cudaStream_t>(stream), nullptr, 0),
                       /*configUnsupported=*/true);
}

int ovrfsr_dispatch_fsr_rcas(const ovrfsr_image *src_tagged, const ovrfsr_image *dst_tagged, const uint32_t consts[12], int math_mode,
                             void *stream) {
  return ovrfsr_dispatch_fsr_rcas_ex(src_tagged, dst_tagged, consts, math_mode, 0, stream);
}

int ovrfsr_dispatch_fsr_rcas_ex(const ovrfsr_image *src_tagged, const ovrfsr_image *dst_tagged, const uint32_t consts[12], int math_mode,
                                int pass_flags, void *stream) {
  const DispatchPair io(src_tagged, dst_tagged);
  const Image *src = io.src, *dst = io.dst;
  if (!consts) return OVRFSR_ERR_INVALID;
  int rc = check_pair(src, dst);
  if (rc != OVRFSR_OK || (rc = check_pass_flags(src, pass_flags)) != OVRFSR_OK) return rc;
  if (src->width != dst->width || src->height != dst->height) return OVRFSR_ERR_INVALID;
  return launch_status(launchers(math_mode).rcas(pass_image(*src), pass_image(*dst), consts, static_cast<cudaStream_t>(stream), false,
                                                 nullptr, pass_flags),
                       /*configUnsupported=*/false);
}

int ovrfsr_dispatch_nis_scaler(const ovrfsr_image *src_tagged, const ovrfsr_image *dst_tagged, const void *cfg256, int math_mode,
                               void *stream) {
  return ovrfsr_dispatch_nis_scaler_ex(src_tagged, dst_tagged, cfg256, math_mode, 0, stream);
}

int ovrfsr_dispatch_nis_sharpen(const ovrfsr_image *src_tagged, const ovrfsr_image *dst_tagged, const void *cfg256, int math_mode,
                                void *stream) {
  return ovrfsr_dispatch_nis_sharpen_ex(src_tagged, dst_tagged, cfg256, math_mode, 0, stream);
}

// NVScaler, or NVSharpen (sharpen), with this library's filter banks
static int dispatch_nis(bool sharpen, const ovrfsr_image *src_tagged, const ovrfsr_image *dst_tagged, const void *cfg256, int math_mode,
                        int pass_flags, void *stream) {
  const DispatchPair io(src_tagged, dst_tagged);
  const Image *src = io.src, *dst = io.dst;
  if (!cfg256) return OVRFSR_ERR_INVALID;
  int rc = check_nis_image(src, false);
  if (rc != OVRFSR_OK || (rc = check_nis_image(dst, true)) != OVRFSR_OK) return rc;
  if ((rc = check_pass_flags(src, pass_flags)) != OVRFSR_OK) return rc;
  if (sharpen && (src->width != dst->width || src->height != dst->height)) return OVRFSR_ERR_INVALID;
  const Launchers &L = launchers(math_mode);
  return launch_status((sharpen ? L.nis_sharpen : L.nis_scaler)(pass_image(*src), pass_image(*dst), cfg256, static_cast<cudaStream_t>(stream),
                                                                nullptr, pass_flags),
                       /*configUnsupported=*/true);
}

int ovrfsr_dispatch_nis_scaler_ex(const ovrfsr_image *src_tagged, const ovrfsr_image *dst_tagged, const void *cfg256, int math_mode,
                                  int pass_flags, void *stream) {
  return dispatch_nis(false, src_tagged, dst_tagged, cfg256, math_mode, pass_flags, stream);
}

int ovrfsr_dispatch_nis_sharpen_ex(const ovrfsr_image *src_tagged, const ovrfsr_image *dst_tagged, const void *cfg256, int math_mode,
                                   int pass_flags, void *stream) {
  return dispatch_nis(true, src_tagged, dst_tagged, cfg256, math_mode, pass_flags, stream);
}

// ---- host constants -----------------------------------------------------------------------------
void ovrfsr_output_size(uint32_t in_w, uint32_t in_h, float render_scale, uint32_t *out_w, uint32_t *out_h) {
  uint32_t w = 0, h = 0;
  host::output_size(in_w, in_h, render_scale, &w, &h);
  if (out_w) *out_w = w;
  if (out_h) *out_h = h;
}
void ovrfsr_fsr_easu_con(uint32_t con[16], float vw, float vh, float iw, float ih, float ow, float oh) {
  host::fsr_easu_con(con, vw, vh, iw, ih, ow, oh);
}
void ovrfsr_fsr_rcas_con(uint32_t con[4], float stops) { host::fsr_rcas_con(con, stops); }
void ovrfsr_make_upscale_constants(uint32_t consts[24], const ovrfsr_config *cfg, int eye, int only_one_eye, uint32_t in_w,
                                   uint32_t in_h, uint32_t out_w, uint32_t out_h) {
  host::make_upscale_constants(consts, *cfg, eye, only_one_eye != 0, in_w, in_h, out_w, out_h);
}
void ovrfsr_make_sharpen_constants(uint32_t consts[12], const ovrfsr_config *cfg, int eye, int only_one_eye, uint32_t out_w,
                                   uint32_t out_h) {
  host::make_sharpen_constants(consts, *cfg, eye, only_one_eye != 0, out_w, out_h);
}

// ---- introspection ------------------------------------------------------------------------------
int ovrfsr_get_upscale_constants(const ovrfsr_ctx *ctx, int eye, uint32_t consts[24]) {
  if (!ctx || !consts || (eye != 0 && eye != 1) || !ctx->initialized) return OVRFSR_ERR_INVALID;
  std::memcpy(consts, ctx->upscaleConstants[ctx->textureContainsOnlyOneEye ? eye : 0], 96);
  return OVRFSR_OK;
}
int ovrfsr_get_sharpen_constants(const ovrfsr_ctx *ctx, int eye, uint32_t consts[12]) {
  if (!ctx || !consts || (eye != 0 && eye != 1) || !ctx->initialized) return OVRFSR_ERR_INVALID;
  std::memcpy(consts, ctx->sharpenConstants[ctx->textureContainsOnlyOneEye ? eye : 0], 48);
  return OVRFSR_OK;
}
void ovrfsr_cas_setup(uint32_t consts[8], float sharpness, float max_color_delta, float in_w, float in_h, float out_w, float out_h) {
  if (consts) host::cas_setup(consts, sharpness, max_color_delta, in_w, in_h, out_w, out_h);
}

int ovrfsr_dispatch_cas(const ovrfsr_image *src_tagged, const ovrfsr_image *dst_tagged, const uint32_t consts[8], int sharpen_only, int math_mode,
                        void *stream) {
  const DispatchPair io(src_tagged, dst_tagged);
  const Image *src = io.src, *dst = io.dst;
  if (!consts) return OVRFSR_ERR_INVALID;
  if (io.any_array()) return OVRFSR_ERR_UNSUPPORTED; /* CAS has no array I/O */
  int rc = check_pair(src, dst);
  if (rc != OVRFSR_OK) return rc;
  return launch_status(launchers(math_mode).cas(pass_image(*src), pass_image(*dst), consts, sharpen_only, static_cast<cudaStream_t>(stream)),
                       /*configUnsupported=*/false);
}

int ovrfsr_selftest_rcp(uint32_t *mismatches, uint32_t *checked) {
  uint32_t r[2] = {0, 0};
  if (selftest_rcas_rcp(r, nullptr) != cudaSuccess) return OVRFSR_ERR_CUDA;
  if (mismatches) *mismatches = r[0];
  if (checked) *checked = r[1];
  return OVRFSR_OK;
}
int ovrfsr_selftest_div(uint32_t *mismatches, uint32_t *checked) {
  uint32_t r[2] = {0, 0};
  if (selftest_nis_div(r, nullptr) != cudaSuccess) return OVRFSR_ERR_CUDA;
  if (mismatches) *mismatches = r[0];
  if (checked) *checked = r[1];
  return OVRFSR_OK;
}
uint64_t ovrfsr_kernel_launches(void) { return ovrfsr::g_launches.load(std::memory_order_relaxed); }

int ovrfsr_get_gpu_time_ms(ovrfsr_ctx *ctx, float *mean_ms) {
  if (!ctx || !mean_ms) return 0;
  harvest_queries(ctx);
  if (ctx->countedQueries == 0) return 0;
  // "Average GPU processing time for upscale", x2 when each texture holds one eye (PostProcessor.cpp:619-626)
  float avg = ctx->summedGpuTime / (float)ctx->countedQueries;
  if (ctx->textureContainsOnlyOneEye) avg *= 2;
  *mean_ms = avg;
  return ctx->countedQueries;
}

const char *ovrfsr_last_error(const ovrfsr_ctx *ctx) { return ctx ? ctx->lastError.c_str() : "null context"; }

const char *ovrfsr_status_string(int status) {
  switch (status) {
    case OVRFSR_OK: return "ok";
    case OVRFSR_ERR_INVALID: return "invalid argument";
    case OVRFSR_ERR_UNSUPPORTED: return "unsupported format or scale";
    case OVRFSR_ERR_CUDA: return "CUDA failure or no device";
    case OVRFSR_ERR_NOMEM: return "out of memory";
    case OVRFSR_PASSTHROUGH: return "post-processing disabled: pass-through";
    default: return "unknown status";
  }
}
uint32_t ovrfsr_version(void) { return OVRFSR_VERSION; }

int ovrfsr_image_alloc(ovrfsr_image *img, uint32_t width, uint32_t height, int32_t format) {
  if (!img || width == 0 || height == 0 || !valid_format(format)) return OVRFSR_ERR_INVALID;
  DeviceImage d;
  if (!d.alloc(width, height, format)) return OVRFSR_ERR_NOMEM;
  *img = d.img;
  return OVRFSR_OK;
}
int ovrfsr_image_alloc_array(ovrfsr_image *img, uint32_t width, uint32_t height, int32_t format, uint32_t layers) {
  if (!img || width == 0 || height == 0 || format < 0) return OVRFSR_ERR_INVALID;
  cudaChannelFormatDesc desc;
  if (!array_channel_desc(format & OVRFSR_FORMAT_LAYOUT_MASK, &desc))
    return valid_format(format & OVRFSR_FORMAT_LAYOUT_MASK) ? OVRFSR_ERR_UNSUPPORTED : OVRFSR_ERR_INVALID;
  const bool layered = layers > 1;
  cudaArray_t a = nullptr;
  const cudaError_t e = cudaMalloc3DArray(&a, &desc, make_cudaExtent(width, height, layered ? layers : 0),
                                          cudaArraySurfaceLoadStore | (layered ? cudaArrayLayered : 0u));
  if (e != cudaSuccess) {
    cudaGetLastError();
    return e == cudaErrorMemoryAllocation ? OVRFSR_ERR_NOMEM : OVRFSR_ERR_CUDA;
  }
  *img = ovrfsr_image{a, width, height, 0, format | OVRFSR_FORMAT_ARRAY_BIT, layered ? layers : 1u, 0, 0};
  return OVRFSR_OK;
}

int ovrfsr_release_array(const ovrfsr_image *img) {
  if (!img || !img->data || !untagged(*img).array) return OVRFSR_ERR_INVALID;
  return release_array_objects(img->data) == cudaSuccess ? OVRFSR_OK : OVRFSR_ERR_CUDA;
}

void ovrfsr_image_free(ovrfsr_image *img) {
  if (img && img->data) {
    if (untagged(*img).array) {
      release_array_objects(img->data);
      cudaFreeArray(static_cast<cudaArray_t>(img->data));
    } else {
      cudaFree(img->data);
    }
  }
  if (img) *img = ovrfsr_image{};
}

int ovrfsr_image_copy(const ovrfsr_image *dst_tagged, const ovrfsr_image *src_tagged, void *stream) {
  if (!dst_tagged || !src_tagged) return OVRFSR_ERR_INVALID;
  const Image src = untagged(*src_tagged), dst = untagged(*dst_tagged);
  int rc = validate_image(&src);
  if (rc != OVRFSR_OK || (rc = validate_image(&dst)) != OVRFSR_OK) return rc;
  const uint32_t slices = src.array_slices > 1 ? src.array_slices : 1u;
  if (src.width != dst.width || src.height != dst.height || src.format != dst.format || slices != (dst.array_slices > 1 ? dst.array_slices : 1u))
    return OVRFSR_ERR_INVALID;
  if (src.sample_count > 1 || dst.sample_count > 1) return OVRFSR_ERR_UNSUPPORTED;
  const size_t rowBytes = (size_t)src.width * bytes_per_pixel(src.format);
  for (uint32_t z = 0; z < slices; ++z) {
    // one slice per copy: pitched slices sit slice_pitch apart, array layers are addressed by z
    cudaMemcpy3DParms p{};
    if (src.array) { p.srcArray = static_cast<cudaArray_t>(src.data); p.srcPos = make_cudaPos(0, 0, slices > 1 ? z : 0); }
    else p.srcPtr = make_cudaPitchedPtr(static_cast<uint8_t *>(src.data) + (size_t)z * src.slice_pitch, src.pitch, rowBytes, src.height);
    if (dst.array) { p.dstArray = static_cast<cudaArray_t>(dst.data); p.dstPos = make_cudaPos(0, 0, slices > 1 ? z : 0); }
    else p.dstPtr = make_cudaPitchedPtr(static_cast<uint8_t *>(dst.data) + (size_t)z * dst.slice_pitch, dst.pitch, rowBytes, dst.height);
    // the extent's width counts elements when an array takes part, bytes otherwise
    p.extent = make_cudaExtent(src.array || dst.array ? src.width : rowBytes, src.height, 1);
    p.kind = cudaMemcpyDeviceToDevice;
    const cudaError_t e = cudaMemcpy3DAsync(&p, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return OVRFSR_ERR_CUDA;
  }
  return OVRFSR_OK;
}

} // extern "C"

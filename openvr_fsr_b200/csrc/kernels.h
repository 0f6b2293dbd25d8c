// kernels.h -- host-visible launchers of the sm_90a kernels, one set per math mode.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ovrfsr.h"

namespace ovrfsr {

// One kernel operand.  ptr is a device pointer with row pitch `pitch`, or, when `array` is set, a cudaArray_t (pitch
// unused; `layer` selects the layer of a layered array, -1 = not layered).
struct PassImage { void *ptr; uint32_t pitch; int w, h; int format; bool array = false; int layer = -1; };

// the `centreDev` block described below: its size in words and where its sharpness words sit
constexpr int kLatchWords = 16, kLatchRcasSharp = 6, kLatchNisSharp = 8;

// FSR (fsr_kernels.cuh).  consts are the reference's constant-buffer layouts.
// `direct` (EASU) / `skipOutside` (RCAS) are the ctx path's pairing of the two passes: when RCAS follows EASU in the same
// apply, EASU writes the outside-radius groups -- which RCAS would only copy (x the debug tint `tintGB`) -- straight
// to the final image `direct`, and RCAS visits only tiles / groups inside the radius.  Same output bits as two plain
// dispatches; a stateless dispatch passes nullptr / false.
// `centreDev` (every masked launcher): nullptr = the mask and sharpness words of the constant block; else a 64-byte
// device block the kernels read those words from when they run (the ctx path with a focus, a focus radius or a
// sharpness override: ovrfsr_set_focus / ovrfsr_set_focus_radius / ovrfsr_set_sharpness):
//   words 0-3 imageCentre, 4-5 radiusSq of centre pair 0 / 1, 6 RCAS const0[0] (RCAS and the fused kernel),
//   8-9 NISConfig kSharpStrengthMin / kSharpStrengthScale, 10-11 kSharpLimitMin / kSharpLimitScale (NVScaler and
//   NVSharpen), 7 and 12-15 padding.  EASU reads words 0-5 only.
// `srtm` (EASU and RCAS): OVRFSR_PASS_SRTM_* bits, AMD's reversible tone map on the texels read / the pixels stored.
// Float sources only, and never together with the pairing: cudaErrorInvalidValue otherwise.
cudaError_t launch_easu_fast(const PassImage &src, const PassImage &dst, const uint32_t consts[24], cudaStream_t s,
                             const PassImage *direct = nullptr, float tintGB = 1.0f, const uint32_t *centreDev = nullptr,
                             int srtm = 0);
cudaError_t launch_easu_strict(const PassImage &src, const PassImage &dst, const uint32_t consts[24], cudaStream_t s,
                               const PassImage *direct = nullptr, float tintGB = 1.0f, const uint32_t *centreDev = nullptr,
                               int srtm = 0);
cudaError_t launch_rcas_fast(const PassImage &src, const PassImage &dst, const uint32_t consts[12], cudaStream_t s,
                             bool skipOutside = false, const uint32_t *centreDev = nullptr, int srtm = 0);
cudaError_t launch_rcas_strict(const PassImage &src, const PassImage &dst, const uint32_t consts[12], cudaStream_t s,
                               bool skipOutside = false, const uint32_t *centreDev = nullptr, int srtm = 0);

// EASU -> RCAS in one kernel (fsr_fused.cuh): ku = UpscaleConstants, ks = SharpenConstants; dst.format (RGBA8, or RGB10A2
// for an RGB10A2 source) is also the format the intermediate is quantised to.  cudaErrorInvalidValue /
// cudaErrorInvalidConfiguration = this pair of passes cannot be fused (the caller runs the two dispatches instead).
cudaError_t launch_fsr_fused_fast(const PassImage &src, const PassImage &dst, const uint32_t ku[24], const uint32_t ks[12], cudaStream_t s,
                                  const uint32_t *centreDev = nullptr);
cudaError_t launch_fsr_fused_strict(const PassImage &src, const PassImage &dst, const uint32_t ku[24], const uint32_t ks[12], cudaStream_t s,
                                    const uint32_t *centreDev = nullptr);

// NIS (nis_kernels.cuh).  cfg = the 256-byte NISConfig block; coef = [2][64][8] floats (scale, usm) on the host.
// `srtm`: OVRFSR_PASS_SRTM_* bits as for EASU and RCAS (OVRFSR_FLAG_SRTM_NIS).  Float sources only: cudaErrorInvalidValue
// otherwise.
cudaError_t launch_nis_scaler_fast(const PassImage &src, const PassImage &dst, const void *cfg256, const float *coef, cudaStream_t s,
                                   const uint32_t *centreDev = nullptr, int srtm = 0);
cudaError_t launch_nis_scaler_strict(const PassImage &src, const PassImage &dst, const void *cfg256, const float *coef, cudaStream_t s,
                                     const uint32_t *centreDev = nullptr, int srtm = 0);
cudaError_t launch_nis_sharpen_fast(const PassImage &src, const PassImage &dst, const void *cfg256, const float *coef, cudaStream_t s,
                                    const uint32_t *centreDev = nullptr, int srtm = 0);
cudaError_t launch_nis_sharpen_strict(const PassImage &src, const PassImage &dst, const void *cfg256, const float *coef, cudaStream_t s,
                                      const uint32_t *centreDev = nullptr, int srtm = 0);
// NVScaler (sharpenOnly false) or NVSharpen with this library's filter banks, on images already validated (nis_capi.cu)
cudaError_t launch_nis(bool sharpenOnly, const PassImage &src, const PassImage &dst, const void *cfg256, int mathMode, cudaStream_t s,
                       const uint32_t *centreDev = nullptr, int srtm = 0);

// legacy CAS (cas_kernels.cuh).  consts = const0, const1 of src/cas/cas.compute.h:1-4 as CasSetup fills them.
cudaError_t launch_cas_fast(const PassImage &src, const PassImage &dst, const uint32_t consts[8], int sharpenOnly, cudaStream_t s);
cudaError_t launch_cas_strict(const PassImage &src, const PassImage &dst, const uint32_t consts[8], int sharpenOnly, cudaStream_t s);

// exhaustive device check of strict RCAS's UNORM8 reciprocal: result = {mismatches, operands checked}
cudaError_t selftest_rcas_rcp(uint32_t result[2], cudaStream_t s);
// strict NIS's in-range IEEE quotient (div_rn_inrange) against div.rn on ~19 M operand pairs: {mismatches, checked}
cudaError_t selftest_nis_div(uint32_t result[2], cudaStream_t s);

// MSAA resolve front-end (GetInputView's ResolveSubresource, PostProcessor.cpp:219-226): dst = mean over the
// `samples` consecutive samples of each texel; same format both sides.  One arithmetic (strict) for both math modes.
cudaError_t launch_resolve_msaa(const PassImage &srcSamples, int samples, const PassImage &dst, cudaStream_t s);

// bumped once per kernel launch by every launcher (ovrfsr_kernel_launches)
void count_launch();

} // namespace ovrfsr

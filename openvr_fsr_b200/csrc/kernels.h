// kernels.h -- host-visible launchers of the sm_90a kernels, one table per math mode.
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

// The per-texel maps of a pass (`maps` below): OVRFSR_PASS_* bits of the texels it reads and of the pixels it stores.
// Read order finite-in, SRTM's F, perceptual P; store order P^-1, G, finite-out or the sRGB encode (device_common.cuh,
// map_in / map_out).  The maps are defined for float sources only.
constexpr int kMapsIn = OVRFSR_PASS_SRTM_IN | OVRFSR_PASS_FINITE_IN | OVRFSR_PASS_PERCEPTUAL_IN;
constexpr int kMapsOut = OVRFSR_PASS_SRTM_OUT | OVRFSR_PASS_FINITE_OUT | OVRFSR_PASS_PERCEPTUAL_OUT;

// The launchers of one math mode, one per pass: kernels_fast.cu fills kFastLaunchers, kernels_strict.cu kStrictLaunchers.
struct Launchers {
  // FSR (fsr_kernels.cuh).  consts are the reference's constant-buffer layouts.
  // `direct` (EASU) / `skipOutside` (RCAS) are the ctx path's pairing of the two passes: when RCAS follows EASU in the
  // same apply, EASU writes the outside-radius groups -- which RCAS would only copy (x the debug tint `tintGB`) --
  // straight to the final image `direct`, and RCAS visits only tiles / groups inside the radius.  Same output bits as
  // two plain dispatches; a stateless dispatch passes nullptr / false.
  // `centreDev` (every masked launcher): nullptr = the mask and sharpness words of the constant block; else a 64-byte
  // device block the kernels read those words from when they run (the ctx path with a focus, a focus radius or a
  // sharpness override: ovrfsr_set_focus / ovrfsr_set_focus_radius / ovrfsr_set_sharpness):
  //   words 0-3 imageCentre, 4-5 radiusSq of centre pair 0 / 1, 6 RCAS const0[0] (RCAS and the fused kernel),
  //   8-9 NISConfig kSharpStrengthMin / kSharpStrengthScale, 10-11 kSharpLimitMin / kSharpLimitScale (NVScaler and
  //   NVSharpen), 7 and 12-15 padding.  EASU reads words 0-5 only.
  // `maps` (every launcher but CAS): kMapsIn | kMapsOut bits.  Any bit with a UNORM source, or a bit the pass does not
  // take, is cudaErrorInvalidValue.  EASU with `direct` takes only the finite bits (finite-out does nothing to its UNORM
  // stores), RCAS with `skipOutside` none: the pairing copies UNORM codes, which mapped values are not.
  cudaError_t (*easu)(const PassImage &src, const PassImage &dst, const uint32_t consts[24], cudaStream_t s,
                      const PassImage *direct, float tintGB, const uint32_t *centreDev, int maps);
  cudaError_t (*rcas)(const PassImage &src, const PassImage &dst, const uint32_t consts[12], cudaStream_t s,
                      bool skipOutside, const uint32_t *centreDev, int maps);
  // EASU -> RCAS in one kernel (fsr_fused.cuh): ku = UpscaleConstants, ks = SharpenConstants; dst.format (RGBA8, or
  // RGB10A2 for an RGB10A2 source) is also the format the intermediate is quantised to.  cudaErrorInvalidValue /
  // cudaErrorInvalidConfiguration = this pair of passes cannot be fused (the caller runs the two dispatches instead).
  // `maps`: the finite bits only; finite-in on every texel read, and finite-out does nothing to the UNORM target.
  cudaError_t (*fsr_fused)(const PassImage &src, const PassImage &dst, const uint32_t ku[24], const uint32_t ks[12],
                           cudaStream_t s, const uint32_t *centreDev, int maps);
  // NIS (nis_kernels.cuh), with this library's filter banks.  cfg256 = the 256-byte NISConfig block.
  cudaError_t (*nis_scaler)(const PassImage &src, const PassImage &dst, const void *cfg256, cudaStream_t s,
                            const uint32_t *centreDev, int maps);
  cudaError_t (*nis_sharpen)(const PassImage &src, const PassImage &dst, const void *cfg256, cudaStream_t s,
                             const uint32_t *centreDev, int maps);
  // legacy CAS (cas_kernels.cuh).  consts = const0, const1 of src/cas/cas.compute.h:1-4 as CasSetup fills them.
  cudaError_t (*cas)(const PassImage &src, const PassImage &dst, const uint32_t consts[8], int sharpenOnly, cudaStream_t s);
};
extern const Launchers kFastLaunchers, kStrictLaunchers;

// the launchers of ovrfsr_config::math_mode / a dispatch's math_mode: strict for OVRFSR_MATH_STRICT, fast otherwise
inline const Launchers &launchers(int mathMode) { return mathMode == OVRFSR_MATH_STRICT ? kStrictLaunchers : kFastLaunchers; }

// exhaustive device check of strict RCAS's UNORM8 reciprocal: result = {mismatches, operands checked}
cudaError_t selftest_rcas_rcp(uint32_t result[2], cudaStream_t s);
// strict NIS's in-range IEEE quotient (div_rn_inrange) against div.rn on ~19 M operand pairs: {mismatches, checked}
cudaError_t selftest_nis_div(uint32_t result[2], cudaStream_t s);

// MSAA resolve front-end (GetInputView's ResolveSubresource, PostProcessor.cpp:219-226): dst = mean over the
// `samples` consecutive samples of each texel; same format both sides.  One arithmetic (strict) for both math modes.
cudaError_t launch_resolve_msaa(const PassImage &srcSamples, int samples, const PassImage &dst, cudaStream_t s);

} // namespace ovrfsr

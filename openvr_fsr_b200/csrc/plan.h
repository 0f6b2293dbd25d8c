// plan.h -- what every apply of a context runs, decided once per prepare_resources (capi.cu).  Host only.
#pragma once

#include "../../include/ovrfsr.h"

namespace ovrfsr {

// What every apply of a context runs (PostProcessor.cpp:586-594), decided by prepare_resources from the config, the
// source format and the output format, none of which can change before the next prepare_resources.  FSR always runs
// RCAS, after EASU when upscaling; NIS runs one pass, NVScaler when upscaling and NVSharpen otherwise.  The last pass
// writes the caller's image or the ctx's output image.
struct Plan {
  bool nis = false;
  bool upscale = false; // render_scale != 1
  // EASU followed by RCAS with a UNORM target: EASU writes the outside-radius groups straight to the final image and
  // RCAS only visits what is inside the radius (kernels.h).  The two passes must classify every group the same way, or
  // a group would be written by neither or filtered twice: with a focus or a radius override both read their centre
  // and radius words from the one device block that the single copy at the head of the apply wrote on the same stream
  // (apply_post_process), so an update that lands between the two launches cannot split them.
  bool paired = false;
  bool tryFused = false;               // paired and OVRFSR_FLAG_FUSED_FSR: one fused kernel, where the images allow it
  int easuMaps = 0, rcasMaps = 0;      // OVRFSR_PASS_* bits of each FSR pass (the fused kernel takes easuMaps)
  int nisMaps = 0;                     // OVRFSR_PASS_* bits of the NIS pass
  int midFormat = OVRFSR_FORMAT_RGBA8; // of FSR's upscaled image
  bool srgbOut = false;                // the last pass sRGB-encodes its UNORM8 store (OVRFSR_FLAG_PERCEPTUAL)
};

inline bool float_source(int format) {
  return format == OVRFSR_FORMAT_RGBA16F || format == OVRFSR_FORMAT_RGBA32F || format == OVRFSR_FORMAT_RGB32F;
}

// OVRFSR_FLAG_PERCEPTUAL with a float source and an RGBA8 output (a float source never gets RGB10A2): the last pass
// stores sRGB codes.  Decided from the config and the source alone, so that apply_impl can judge a destination's tag
// before prepare_resources runs.
inline bool srgb_output(const ovrfsr_config &cfg, int srcFormat) {
  return (cfg.flags & OVRFSR_FLAG_PERCEPTUAL) && float_source(srcFormat) &&
         (cfg.output_format == OVRFSR_FORMAT_AUTO || cfg.output_format == OVRFSR_FORMAT_RGBA8);
}

// The plan of a config, a source format and the output format prepare_resources accepted for them (DESIGN.md §3,
// "The per-texel maps of a pass").  The maps take effect with a float source (an RGB32F one is read through its RGBA32F
// copy, a multisampled one after its resolve); UNORM sources are display-referred already and get no bits.
inline Plan make_plan(const ovrfsr_config &cfg, int srcFormat, int outFormat) {
  Plan p;
  p.nis = cfg.use_nis != 0;
  p.upscale = cfg.render_scale != 1.f;
  const bool floatSrc = float_source(srcFormat);
  const bool tone = floatSrc && (cfg.flags & (p.nis ? OVRFSR_FLAG_SRTM_NIS : OVRFSR_FLAG_SRTM));
  const bool perceptual = floatSrc && (cfg.flags & OVRFSR_FLAG_PERCEPTUAL);
  // the first pass maps every texel it reads, the last pass maps back every pixel it stores
  const int in = (tone ? OVRFSR_PASS_SRTM_IN : 0) | (perceptual ? OVRFSR_PASS_PERCEPTUAL_IN : 0);
  const int out = (tone ? OVRFSR_PASS_SRTM_OUT : 0) | (perceptual ? OVRFSR_PASS_PERCEPTUAL_OUT : 0);
  // Mapped values are neither the eye's UNORM codes, which the pairing copies, nor fit for a UNORM intermediate: RCAS's
  // G amplifies tone-mapped values by up to 32768 near 1 and P^-1 squares perceptual ones, so the intermediate keeps
  // them as RGBA32F for a float output and as RGBA16F for a UNORM output, which clips at 1 anyway (an RGBA8
  // intermediate would band).
  const bool unormOut = outFormat == OVRFSR_FORMAT_RGBA8 || outFormat == OVRFSR_FORMAT_RGB10A2;
  p.paired = !p.nis && p.upscale && unormOut && !(tone || perceptual);
  p.tryFused = p.paired && (cfg.flags & OVRFSR_FLAG_FUSED_FSR);
  p.midFormat = !(tone || perceptual) ? outFormat : (unormOut ? OVRFSR_FORMAT_RGBA16F : OVRFSR_FORMAT_RGBA32F);
  p.srgbOut = srgb_output(cfg, srcFormat);
  // OVRFSR_FLAG_FINITE on every pass that reads a float image: finite-in on what it reads, finite-out on what it stores
  // (a UNORM store ignores it).  After EASU only the paired RCAS reads a UNORM intermediate.
  const int finite = floatSrc && (cfg.flags & OVRFSR_FLAG_FINITE) ? OVRFSR_PASS_FINITE_IN | OVRFSR_PASS_FINITE_OUT : 0;
  if (p.nis) {
    p.nisMaps = in | out | finite;
  } else if (p.upscale) {
    p.easuMaps = in | finite;
    p.rcasMaps = out | (p.paired ? 0 : finite);
  } else {
    p.rcasMaps = in | out | finite;
  }
  return p;
}

} // namespace ovrfsr

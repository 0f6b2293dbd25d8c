// config.h -- the process-wide Config singleton the hook layer reads
// (/root/reference/src/postprocess/Config.h:10-28,65-68), reduced to the fields that steer this path.
// Loading openvr_mod.cfg (jsoncpp, Win32 paths) stays with the mod; whoever owns the file fills this in.
#pragma once

#include "../../include/ovrfsr.h"

struct Config {
  bool fsrEnabled = false;
  bool applyMIPBias = true; // consumed by the D3D11 sampler hook (VrHooks.cpp:94-136), not by this path
  float renderScale = 1.f;
  float sharpness = 0.75f;
  float radius = 0.5f;
  bool debugMode = false;
  bool useNis = false;
  // not in the reference's Config: what it queries from the live runtime / picks implicitly
  float projCentre[4] = {0.5f, 0.5f, 0.5f, 0.5f}; // CalculateProjectionCenter, PostProcessor.cpp:104-121
  int cudaDevice = -1;
  bool strictMath = true;   // bit-identical to the reference lines (the library default); false = FMA-contracted kernels, <= 1 LSB per pass
  bool fusedFsr = false;    // OVRFSR_FLAG_FUSED_FSR: one fused EASU->RCAS kernel instead of the two dispatches
  bool srtm = false;        // OVRFSR_FLAG_SRTM: FSR on a float (HDR) eye texture runs inside AMD's reversible tone map
  bool srtmNis = false;     // OVRFSR_FLAG_SRTM_NIS: NIS on a float (HDR) eye texture runs inside the same tone map
  bool finite = false;      // OVRFSR_FLAG_FINITE: no infinity or NaN of a float eye texture enters a pass or a stored pixel
  bool perceptual = false;  // OVRFSR_FLAG_PERCEPTUAL: a float eye texture is filtered as gamma 2.0, an 8-bit output is sRGB

  // ONE instance per process, owned by libovrfsr.so (an inline function-local static would be duplicated in every
  // module that includes this header when the library is built with hidden visibility)
  OVRFSR_API static Config &Instance();
};

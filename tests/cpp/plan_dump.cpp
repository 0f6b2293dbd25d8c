// plan_dump.cpp -- prints make_plan (csrc/plan.h) for every use_nis, render scale 1 / 0.75, ovrfsr_config::output_format,
// source format and flags 0..31, one line each:
//   use_nis upscale cfg_output_format src_format flags out_format paired tryFused midFormat srgbOut easu rcas nis
// out_format is DetermineOutputFormat's (prepare_resources), whether or not prepare_resources accepts it.
// Built and run by tests/test_plan_host.py with a plain host compiler.
#include <cstdio>

#include "plan.h"

int main() {
  const float scales[] = {1.0f, 0.75f};
  const int cfgOuts[] = {OVRFSR_FORMAT_AUTO, OVRFSR_FORMAT_RGBA8, OVRFSR_FORMAT_RGB10A2, OVRFSR_FORMAT_RGBA16F,
                         OVRFSR_FORMAT_RGBA32F};
  for (int nis = 0; nis < 2; ++nis)
    for (float scale : scales)
      for (int cfgOut : cfgOuts)
        for (int src = OVRFSR_FORMAT_RGBA8; src <= OVRFSR_FORMAT_RGB32F; ++src)
          for (int flags = 0; flags < 32; ++flags) {
            ovrfsr_config cfg{};
            cfg.use_nis = nis;
            cfg.render_scale = scale;
            cfg.output_format = cfgOut;
            cfg.flags = flags;
            const int out = cfgOut != OVRFSR_FORMAT_AUTO ? cfgOut
                            : src == OVRFSR_FORMAT_RGB10A2 ? OVRFSR_FORMAT_RGB10A2 : OVRFSR_FORMAT_RGBA8;
            const ovrfsr::Plan p = ovrfsr::make_plan(cfg, src, out);
            std::printf("%d %d %d %d %d %d %d %d %d %d %d %d %d\n", nis, scale != 1.0f, cfgOut, src, flags, out, p.paired,
                        p.tryFused, p.midFormat, p.srgbOut, p.easuMaps, p.rcasMaps, p.nisMaps);
          }
  return 0;
}

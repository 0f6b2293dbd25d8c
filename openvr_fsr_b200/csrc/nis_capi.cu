// nis_capi.cu -- NIS half of include/ovrfsr.h: NISConfig setup and the filter banks.
#include <cstring>

#include "nis_host.h"
#include "nis_coef_table.inc"

using namespace ovrfsr;

const float *ovrfsr::host::nis_coef_banks() {
  struct Banks { float bank[2][64 * 8]; };
  static const Banks b = [] {
    Banks r{};
    for (int p = 0; p < 64; ++p)
      for (int t = 0; t < 6; ++t) {
        r.bank[0][p * 8 + t] = (float)(kNisCoefScale1e4[p][t] / 10000.0);
        r.bank[1][p * 8 + t] = (float)(kNisCoefUsm1e4[p][t] / 10000.0);
      }
    return r;
  }();
  return &b.bank[0][0];
}

extern "C" {

int ovrfsr_make_nis_config(void *cfg256, const ovrfsr_config *cfg, int sharpen_only, int eye, int only_one_eye,
                           uint32_t in_w, uint32_t in_h, uint32_t out_w, uint32_t out_h) {
  if (!cfg256 || !cfg) return 0;
  host::NisConfig c;
  const bool ok = host::make_nis_config(c, *cfg, sharpen_only != 0, eye, only_one_eye != 0, in_w, in_h, out_w, out_h);
  std::memcpy(cfg256, &c, sizeof(c));
  return ok ? 1 : 0;
}

const float *ovrfsr_nis_coef_scale(void) { return host::nis_coef_banks(); }
const float *ovrfsr_nis_coef_usm(void) { return host::nis_coef_banks() + 64 * 8; }

} // extern "C"

// minmax_probe.cu -- what sm_90a's fminf / fmaxf / __saturatef return on signed zeros, subnormals, large finite values,
// infinities and NaNs (quiet and signalling, with payloads, of both signs), in the two-operand form and in the nested forms the filters use.  tests/test_gpu_minmax_rule.py builds it
// twice (-fmad=false / -fmad=true), runs each build once and compares every line with the checker's helpers.
//
// The operands are read from device memory, so nothing is folded at compile time: each result is what FMNMX (and the
// saturate modifier) computes.  Output: one line per result, "<form> <operand indices...> <result bits in hex>".
#include <cstdint>
#include <cstdio>
#include <cstring>

#include <cuda_runtime.h>

// {+0, -0, +1, -1, +2^-149, -2^-149, +65504, -65504, NaN, +inf, -inf, signalling NaNs 0x7f800001 / 0xff800001, quiet
// NaNs with a payload 0x7fc00001 / with the sign 0xffc00000}: an FP32 eye texture can hold any of them, and RCAS feeds
// the raw texel to FMNMX
static const uint32_t kValues[] = {0x00000000u, 0x80000000u, 0x3f800000u, 0xbf800000u, 0x00000001u,
                                   0x80000001u, 0x477fe000u, 0xc77fe000u, 0x7fc00000u, 0x7f800000u,
                                   0xff800000u, 0x7f800001u, 0xff800001u, 0x7fc00001u, 0xffc00000u};
constexpr int N = sizeof(kValues) / sizeof(kValues[0]);

// forms, by index into the operand table:
//   min2 / max2 (a, b)                       every ordered pair
//   sat (a)                                  __saturatef(a): FADD.SAT
//   satmul (a, b)                            __saturatef(a * b): FMUL.SAT, how the kernels saturate products
//   satfma (a, b, c)                         __saturatef(fmaf(a, b, c)): FFMA.SAT, saturated sums in fast math
//   min4 / max4 (f, g, j, k)                 fminf(fminf(f, fminf(g, j)), k): EASU's de-ring set, RCAS's ring
//   min3l / max3l (a, b, c)                  fminf(fminf(a, b), c): NIS's contrast ranges
//   min3r / max3r (a, b, c)                  fminf(a, fminf(b, c)): CAS's AMin3F1 / AMax3F1
//   clamp (mn, mx, v)                        fminf(mx, fmaxf(mn, v)): EASU's de-ring clamp, NIS's limit
//   lobe (a, b, c)                           fmaxf(-0.1875, fminf(fmaxf(a, fmaxf(b, c)), 0)): RCAS's lobe
__global__ void probe_pairs(const float *__restrict__ v, float *__restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= N * N) return;
  const float a = v[t / N], b = v[t % N];
  out[2 * t] = fminf(a, b);
  out[2 * t + 1] = fmaxf(a, b);
}
__global__ void probe_sat(const float *__restrict__ v, float *__restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < N) out[t] = __saturatef(v[t]);
}
__global__ void probe_sat_forms(const float *__restrict__ v, float *__restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < N * N) out[t] = __saturatef(v[t / N] * v[t % N]);
  if (t < N * N * N) out[N * N + t] = __saturatef(__fmaf_rn(v[t / (N * N)], v[(t / N) % N], v[t % N]));
}
__global__ void probe_triples(const float *__restrict__ v, float *__restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= N * N * N) return;
  const float a = v[t / (N * N)], b = v[(t / N) % N], c = v[t % N];
  out[6 * t] = fminf(fminf(a, b), c);
  out[6 * t + 1] = fmaxf(fmaxf(a, b), c);
  out[6 * t + 2] = fminf(a, fminf(b, c));
  out[6 * t + 3] = fmaxf(a, fmaxf(b, c));
  out[6 * t + 4] = fminf(b, fmaxf(a, c));
  out[6 * t + 5] = fmaxf(-0.1875f, fminf(fmaxf(a, fmaxf(b, c)), 0.0f));
}
__global__ void probe_quads(const float *__restrict__ v, float *__restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= N * N * N * N) return;
  const float f = v[t / (N * N * N)], g = v[(t / (N * N)) % N], j = v[(t / N) % N], k = v[t % N];
  out[2 * t] = fminf(fminf(f, fminf(g, j)), k);
  out[2 * t + 1] = fmaxf(fmaxf(f, fmaxf(g, j)), k);
}

static int check(cudaError_t e, const char *what) {
  if (e != cudaSuccess) {
    fprintf(stderr, "%s: %s\n", what, cudaGetErrorString(e));
    return 1;
  }
  return 0;
}
static uint32_t bits(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}

int main() {
  constexpr int kPairs = N * N, kTriples = N * N * N, kQuads = N * N * N * N;
  constexpr int kOut = 2 * kPairs + N + 6 * kTriples + 2 * kQuads + kPairs + kTriples;
  float *dv = nullptr, *dout = nullptr;
  static float host[kOut];
  if (check(cudaMalloc(&dv, sizeof(kValues)), "cudaMalloc") || check(cudaMalloc(&dout, sizeof(host)), "cudaMalloc") ||
      check(cudaMemcpy(dv, kValues, sizeof(kValues), cudaMemcpyHostToDevice), "cudaMemcpy"))
    return 1;
  float *oPairs = dout, *oSat = oPairs + 2 * kPairs, *oTriples = oSat + N, *oQuads = oTriples + 6 * kTriples,
        *oSatForms = oQuads + 2 * kQuads;
  probe_pairs<<<(kPairs + 127) / 128, 128>>>(dv, oPairs);
  probe_sat<<<1, 32>>>(dv, oSat);
  probe_triples<<<(kTriples + 255) / 256, 256>>>(dv, oTriples);
  probe_quads<<<(kQuads + 255) / 256, 256>>>(dv, oQuads);
  probe_sat_forms<<<(kTriples + 255) / 256, 256>>>(dv, oSatForms);
  if (check(cudaGetLastError(), "launch") || check(cudaMemcpy(host, dout, sizeof(host), cudaMemcpyDeviceToHost), "cudaMemcpy"))
    return 1;
  cudaFree(dv);
  cudaFree(dout);
  // the same offsets into the host copy
  oPairs = host;
  oSat = oPairs + 2 * kPairs;
  oTriples = oSat + N;
  oQuads = oTriples + 6 * kTriples;
  oSatForms = oQuads + 2 * kQuads;

  for (int t = 0; t < kPairs; ++t) {
    printf("min2 %d %d %08x\n", t / N, t % N, bits(oPairs[2 * t]));
    printf("max2 %d %d %08x\n", t / N, t % N, bits(oPairs[2 * t + 1]));
  }
  for (int t = 0; t < N; ++t) printf("sat %d %08x\n", t, bits(oSat[t]));
  static const char *const kTripleForms[6] = {"min3l", "max3l", "min3r", "max3r", "clamp", "lobe"};
  for (int t = 0; t < kTriples; ++t)
    for (int f = 0; f < 6; ++f)
      printf("%s %d %d %d %08x\n", kTripleForms[f], t / (N * N), (t / N) % N, t % N, bits(oTriples[6 * t + f]));
  for (int t = 0; t < kQuads; ++t) {
    printf("min4 %d %d %d %d %08x\n", t / (N * N * N), (t / (N * N)) % N, (t / N) % N, t % N, bits(oQuads[2 * t]));
    printf("max4 %d %d %d %d %08x\n", t / (N * N * N), (t / (N * N)) % N, (t / N) % N, t % N, bits(oQuads[2 * t + 1]));
  }
  for (int t = 0; t < kPairs; ++t) printf("satmul %d %d %08x\n", t / N, t % N, bits(oSatForms[t]));
  for (int t = 0; t < kTriples; ++t)
    printf("satfma %d %d %d %08x\n", t / (N * N), (t / N) % N, t % N, bits(oSatForms[kPairs + t]));
  return 0;
}

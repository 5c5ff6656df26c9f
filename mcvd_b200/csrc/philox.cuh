// Counter-based noise shared by every op that draws in-kernel (DIFFUSION_UPDATE, NOISE, DSM_PERTURB): Philox4x32-10,
// its Box-Muller normal and the cancellation-free centred Gamma draw.  A draw is keyed by (seed, global clip id,
// step tag, element), so a clip sees the same noise whichever batch position or GPU it lands on.
#pragma once

#include <stdint.h>

namespace mcvd {

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                              uint32_t k1, uint32_t out[4]) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += W0; k1 += W1;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

__device__ __forceinline__ float philox_normal(uint32_t seed_lo, uint32_t seed_hi, uint32_t clip, uint32_t step,
                                               uint32_t elem) {
  uint32_t r[4];
  philox4x32_10(elem, clip, step, 0x4d435644u /* 'MCVD' */, seed_lo, seed_hi, r);
  // Box-Muller on two 32-bit uniforms in (0,1]
  float u1 = ((float)r[0] + 1.0f) * 2.3283064365386963e-10f;
  float u2 = ((float)r[1] + 0.5f) * 2.3283064365386963e-10f;
  u1 = fminf(fmaxf(u1, 1e-12f), 1.0f);
  float rad = sqrtf(-2.0f * logf(u1));
  return rad * cospif(2.0f * u2);
}

// Gamma(k, 1) - k from the same Philox stream (Marsaglia & Tsang 2000, "A simple method for generating gamma
// variables"): d = k - 1/3, c = 1/sqrt(9d), x ~ N(0,1), v = (1 + cx)^3, accept when log u < x^2/2 + d - dv + d log v.
// Attempt a is one Philox call with counter (element, clip, step, MCVD_GAMMA_TAG | a): words 0 and 1 feed Box-Muller,
// word 2 is u, word 3 the boost uniform for k < 1 (G(k) = G(k+1) * U^(1/k)).  Acceptance is >= 0.95 for every
// d >= 2/3, so MCVD_GAMMA_ATTEMPTS = 16 rejections in a row happen with probability < 1e-20 per element; if they do,
// the element takes the proposal's centre v = 1 (x = 0), i.e. G = d.
// k reaches 2.5e10 on the linear schedule, so G - k is never formed as a difference of two large numbers:
// with w = v - 1 = cx(3 + 3cx + c^2x^2), G - k = d w - 1/3 for k >= 1.  Everything runs in fp64; the caller
// rounds to fp32 once.  oracle/gamma_oracle.py restates this function in numpy for the tests.
#define MCVD_GAMMA_TAG 0x47414d00u      /* 'GAM\0' | attempt; distinct from the normal stream's 'MCVD' */
#define MCVD_GAMMA_ATTEMPTS 16

static __device__ __noinline__ double philox_gamma_centred(double k, uint32_t seed_lo, uint32_t seed_hi, uint32_t clip,
                                                           uint32_t step, uint32_t elem) {
  const bool boost = k < 1.0;
  const double kk = boost ? k + 1.0 : k;
  const double d = kk - 1.0 / 3.0, c = 1.0 / sqrt(9.0 * d);
  double w = 0.0, ub = 0.5;
  for (int a = 0; a < MCVD_GAMMA_ATTEMPTS; ++a) {
    uint32_t r[4];
    philox4x32_10(elem, clip, step, MCVD_GAMMA_TAG | (uint32_t)a, seed_lo, seed_hi, r);
    const double u1 = ((double)r[0] + 1.0) * 2.3283064365386963e-10;     // (0, 1]
    const double u2 = ((double)r[1] + 0.5) * 2.3283064365386963e-10;
    const double x = sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);
    const double cx = c * x;
    ub = ((double)r[3] + 0.5) * 2.3283064365386963e-10;
    if (cx <= -1.0) continue;                                              // v <= 0
    const double wc = cx * (3.0 + cx * (3.0 + cx));
    const double u = ((double)r[2] + 0.5) * 2.3283064365386963e-10;
    if (log(u) < 0.5 * x * x + d * (log1p(wc) - wc)) { w = wc; break; }
  }
  if (!boost) return d * w - 1.0 / 3.0;
  return d * (1.0 + w) * exp(log(ub) / k) - k;
}

}  // namespace mcvd

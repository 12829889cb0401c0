// fp8_e4m3.cuh — the operand rule of the opt-in fp8 inference numerics (mpn_ctx_set_option "fp8"), shared by the device
// kernels (fp8.cu: activation and weight quantizers; conv_simt.cu: the check kernel's decode) and the host view
// mpn_debug_fp8 that the CPU suite runs against torch.float8_e4m3fn.
//
// An operand h (the bf16 hi plane of a stored activation or weight) becomes q = rn_e4m3(2^e * h), e4m3 "fn" encoding
// (no infinities, 448 the largest finite value), rounded to nearest even. e is chosen per sample (activations) or per
// output channel (weights) from amax = max |h| over that group:
//   e = the largest integer with amax * 2^e <= 448, clamped to [-60, 60]; amax = 0 gives e = 0.
// So 2^e * h never exceeds 448 and the conversion never saturates. A group whose amax is not finite, or so large that the
// clamp leaves amax * 2^-60 > 448, has no valid scale (scale_ok): the caller fails the call.
// Everything here is bit arithmetic plus one rintf (round half to even in the default rounding mode), so host and device
// give the same bits.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define MPN_FP8_HD __host__ __device__ __forceinline__
#else
#define MPN_FP8_HD inline
#endif

namespace mpn_fp8 {

constexpr int kEmin = -60, kEmax = 60;

MPN_FP8_HD uint32_t f2u(float x) { uint32_t u; memcpy(&u, &x, 4); return u; }
MPN_FP8_HD float u2f(uint32_t u) { float x; memcpy(&x, &u, 4); return x; }
MPN_FP8_HD float pow2(int e) { return u2f((uint32_t)(127 + e) << 23); }      // exact for e in [-126, 127]

// the scale exponent of a group with amax = max |h| (>= 0)
MPN_FP8_HD int scale_exponent(float amax) {
  if (!(amax > 0.f)) return 0;                       // 0 (and NaN: scale_ok rejects it)
  const uint32_t u = f2u(amax);
  const int E = (int)(u >> 23);
  if (E == 255) return 0;                            // inf: scale_ok rejects it
  if (E == 0) return kEmax;                          // fp32 subnormal: far below 448 * 2^-60
  // amax = f * 2^k with f = 1.m / 2 in [0.5, 1), k = E - 126; f * 2^9 <= 448 exactly when 1.m <= 1.75
  const int k = E - 126;
  const int e = ((u & 0x7fffffu) <= 0x600000u ? 9 : 8) - k;
  return e < kEmin ? kEmin : (e > kEmax ? kEmax : e);
}

// amax is finite and amax * 2^e fits e4m3 (false only for non-finite amax, or amax > 448 * 2^60 at the clamp)
MPN_FP8_HD bool scale_ok(float amax, int e) {
  if (!(amax <= 3.4028234663852886e38f)) return false;    // NaN or inf
  return amax * pow2(e) <= 448.f;
}

// rn_e4m3 of a finite x with |x| <= 448: the e4m3fn code (sign bit 0x80; -0 and negative values that round to 0 keep it)
MPN_FP8_HD uint8_t e4m3_rn(float x) {
  const uint32_t u = f2u(x);
  const uint32_t sign = (u >> 24) & 0x80u, a = u & 0x7fffffffu;
  uint32_t code;
  if (a < 0x3c800000u) {                             // |x| < 2^-6: the subnormal grid 2^-9 (code 8 = 2^-6, the smallest normal)
    code = (uint32_t)rintf(u2f(a) * 512.f);
  } else {                                           // keep 3 mantissa bits, half to even; a carry moves into the exponent
    code = ((a + 0x7ffffu + ((a >> 20) & 1u)) >> 20) - ((127u - 7u) << 3);
  }
  return (uint8_t)(sign | code);
}

// the value of an e4m3fn code (never 0x7f / 0xff: e4m3_rn does not produce NaN)
MPN_FP8_HD float e4m3_value(uint8_t q) {
  const int e = (q >> 3) & 15, m = q & 7;
  const float v = e ? (float)(8 + m) * pow2(e - 10) : (float)m * pow2(-9);
  return (q & 0x80) ? -v : v;
}

}  // namespace mpn_fp8

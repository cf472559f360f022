// TEST INFRASTRUCTURE: the arguments and the per-chunk hash of the scalar-math sweep, shared by the host generator of the expected
// hashes (tests/golden/gen_libm_sweep.cpp, which evaluates the ORACLE), the host powf equivalence test (tests/cpp/libm_equiv_pow.cpp)
// and the device probe (tools/probe/libm_sweep_probe.cu, which evaluates the PRODUCT, compiled by nvcc and by NVRTC). Neither the
// product's nor the oracle's math is in here, only which arguments argument index i stands for.
//
// Functions, in the fixture's order. The unary ones take argument i = the f32 with bit pattern i, i < 2^32. The powf sets are 2^28 pairs:
//   pow_x    x = pattern (i >> 5) * 512 + a hashed low 9 bits (every 512th pattern), y = one of the 32 values of SWEEP_Y[i & 31];
//   pow_y    y likewise over every 512th pattern, x = one of the 32 values of SWEEP_X[i & 31];
//   pow_rand two hashed 32-bit patterns; on odd i, y's exponent is folded into [2^-4, 2^4) so that most results are finite.
// Chunks are 2^24 consecutive indices: 256 per unary function, 16 per powf set. A chunk's hash is
//   sum over its i of splitmix64((i << 32) | canon(bits(f(x_i)))) mod 2^64,
// which does not depend on the order of evaluation; canon maps every NaN to 0x7fc00000 and keeps every other pattern (both zeros).
#pragma once
#if defined(__CUDACC__)
#define SWEEP_HD __host__ __device__ __forceinline__
#else
#define SWEEP_HD static inline
#endif
#ifndef __CUDACC_RTC__
#include <cstdint>
#endif

namespace sweep {

enum { SINF, COSF, TANF, TANHF, EXPM1F, EXPF, ATANF, WIDE_SINF, WIDE_ATANF, POW_X, POW_Y, POW_RAND, NFN };
#define SWEEP_NAMES {"sinf", "cosf", "tanf", "tanhf", "expm1f", "expf", "atanf", "wide_sinf", "wide_atanf", "pow_x", "pow_y", "pow_rand"}
constexpr int CHUNK_LOG2 = 24;
SWEEP_HD int chunks(int fn) { return fn >= POW_X ? 16 : 256; }

SWEEP_HD uint64_t splitmix64(uint64_t z) {
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}
SWEEP_HD uint32_t canon(uint32_t b) { return (b & 0x7fffffffu) > 0x7f800000u ? 0x7fc00000u : b; }
SWEEP_HD uint64_t term(uint64_t i, uint32_t result_bits) { return splitmix64((i << 32) | canon(result_bits)); }

// y values against every 512th x: zeros, halves, small integers both signs, 1/3, odd and even integers at 2^24, infinities, NaN,
// the smallest subnormal, 1 +- 1 ulp, large and non-integer values
SWEEP_HD uint32_t y_bits(int k) {
  const uint32_t Y[32] = {0x00000000u, 0x80000000u, 0x3f000000u, 0xbf000000u, 0x3f800000u, 0xbf800000u, 0x40000000u, 0xc0000000u,
                          0x40400000u, 0xc0400000u, 0x3eaaaaabu, 0xbeaaaaabu, 0x4b7fffffu, 0x4b800001u, 0xcb7fffffu, 0x4b800000u,
                          0x7f800000u, 0xff800000u, 0x7fc00000u, 0x00000001u, 0x80000001u, 0x3f800001u, 0x3f7fffffu, 0xbf800001u,
                          0x3fc00000u, 0xbfc00000u, 0x4e000000u, 0x3dcccccdu, 0x42c80000u, 0xc2c80000u, 0x42ff0000u, 0xc3160000u};
  return Y[k];
}
// x values against every 512th y: zeros, +-1 (1 ** NaN, -1 ** +-inf), halves, small integers, 1 +- 1 ulp on both signs, infinities,
// NaN, the smallest subnormal and normal, the largest finite, and values whose powers overflow or underflow early
SWEEP_HD uint32_t x_bits(int k) {
  const uint32_t X[32] = {0x00000000u, 0x80000000u, 0x3f800000u, 0xbf800000u, 0x3f000000u, 0xbf000000u, 0x40000000u, 0xc0000000u,
                          0x40400000u, 0xc0400000u, 0x3f800001u, 0x3f7fffffu, 0xbf800001u, 0xbf7fffffu, 0x7f800000u, 0xff800000u,
                          0x7fc00000u, 0x00000001u, 0x80000001u, 0x00800000u, 0x7f7fffffu, 0xff7fffffu, 0x41200000u, 0xc1200000u,
                          0x3dcccccdu, 0x3eaaaaabu, 0xc1000000u, 0x40e00000u, 0x3f7fbe77u, 0x3f800347u, 0x0da24260u, 0x5f800000u};
  return X[k];
}
SWEEP_HD uint32_t stride_pattern(uint64_t i) {   // every 512th pattern, with hashed low bits so that odd mantissas occur too
  const uint32_t j = (uint32_t)(i >> 5);
  return (j << 9) | (uint32_t)(splitmix64(j) & 0x1ffu);
}
// bit patterns of the arguments of function fn at index i (y only for the powf sets)
SWEEP_HD void arg_bits(int fn, uint64_t i, uint32_t& x, uint32_t& y) {
  if (fn == POW_X) { x = stride_pattern(i); y = y_bits((int)(i & 31)); }
  else if (fn == POW_Y) { x = x_bits((int)(i & 31)); y = stride_pattern(i); }
  else if (fn == POW_RAND) {
    const uint64_t h = splitmix64(i ^ 0x706f77665f72616eull);
    x = (uint32_t)h; y = (uint32_t)(h >> 32);
    if (i & 1) y = (y & 0x807fffffu) | ((123u + ((y >> 23) & 7u)) << 23);
  } else { x = (uint32_t)i; y = 0u; }
}

}  // namespace sweep

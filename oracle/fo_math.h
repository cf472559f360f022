// ORACLE — TEST INFRASTRUCTURE ONLY. Never linked, imported or executed by the product path
// (fundsp_b200/); only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// --impl reference legs may use it, and only as the checker / timed CPU baseline.
//
// CPU restatement of the scalar math substrate of SamiPerttu/fundsp v0.23.0.
// Each function cites the reference file:line it follows (paths relative to the reference crate (SamiPerttu/fundsp v0.23.0)).
//
// PARITY STATUS: integer paths (rnd1, AttoHash, hash32x) are fully in-repo in the reference and
// are pinned bit-for-bit by the golden vectors in tests/golden/. Transcendentals are NOT pinned at
// the ulp level: the reference calls the Rust `libm 0.2.15` crate (musl port) for scalars and
// `wide 1.1.1` for the f32x8 block path; neither source is in the reference crate and no Rust
// toolchain exists here. Scalars are musl's algorithms restated in fo_libm.h (no platform libm on an f32 trig path);
// `wide::f32x8::sin` is restated from its published algorithm (Agner Fog VCL sincos, Cephes
// coefficients) below. "parity unpinned" at ulp level for sin/tan/tanh/exp and wavetable entries.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace fo {

constexpr int MAX_BUFFER_SIZE = 64;  // src/lib.rs:45-48
constexpr int SIMD_N = 8;            // src/lib.rs:61-64
constexpr double DEFAULT_SR = 44100.0;  // src/lib.rs:42

// ---- src/math.rs:569-576 rnd1: SplitMix-style indexed RNG, returns f64 in 0...1.
inline double rnd1(uint64_t x) {
  x ^= 0x5555555555555555ull;
  x *= 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  x = x ^ (x >> 31);
  return (double)(x >> 11) * (1.0 / (double)(1ull << 53));
}

// ---- src/math.rs:589-597 hash1
inline uint64_t hash1(uint64_t x) {
  x ^= 0x5555555555555555ull;
  x *= 0x517cc1b727220a95ull;
  x = (x ^ (x >> 32)) * 0xd6e8feb86659fd93ull;
  x = (x ^ (x >> 32)) * 0xd6e8feb86659fd93ull;
  return x ^ (x >> 32);
}

// ---- src/math.rs:632-658 AttoHash (FxHasher step)
struct AttoHash {
  uint64_t state;
  explicit AttoHash(uint64_t seed = 0) : state(seed) {}
  AttoHash hash(uint64_t data) const {
    uint64_t r = (state << 5) | (state >> 59);
    return AttoHash((r ^ data) * 0x517cc1b727220a95ull);
  }
};

// ---- src/noise.rs:150-157 hash32x
inline uint32_t hash32x(uint32_t x) {
  const uint32_t M = 0x45d9f3bu;
  x = (x ^ (x >> 16)) * M;
  x = (x ^ (x >> 16)) * M;
  return (x ^ (x >> 16)) * M;
}

// Rust f32::max / f32::min semantics (NaN-ignoring) == fmaxf/fminf.
inline float fmax_(float a, float b) { return fmaxf(a, b); }
inline float fmin_(float a, float b) { return fminf(a, b); }

// ---- src/math.rs:129-144 clamp / clamp01 / clamp11 : x.max(lo).min(hi)
template <class T> inline T clampT(T lo, T hi, T x) { return std::fmin(std::fmax(x, lo), hi); }
inline float clamp01f(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }
inline float clamp11f(float x) { return fminf(fmaxf(x, -1.0f), 1.0f); }
inline double clamp01d(double x) { return fmin(fmax(x, 0.0), 1.0); }

// ---- src/math.rs:170-177 Lerp: self * (1 - t) + other * t
inline float lerpf(float a, float b, float t) { return a * (1.0f - t) + b * t; }
inline double lerpd(double a, double b, double t) { return a * (1.0 - t) + b * t; }
// ---- src/math.rs:216-218 delerp
inline float delerpf(float a, float b, float x) { return (x - a) / (b - a); }
inline double delerpd(double a, double b, double x) { return (x - a) / (b - a); }
// ---- src/math.rs:236-238 xerp
inline float xerpf(float a, float b, float t) { return expf(lerpf(logf(a), logf(b), t)); }
inline double xerpd(double a, double b, double t) { return exp(lerpd(log(a), log(b), t)); }
// ---- src/math.rs:415-417 smooth5, :430-437 smooth9
inline double smooth5d(double x) { return ((x * 6.0 - 15.0) * x + 10.0) * x * x * x; }
inline float smooth9f(float x) {
  float x2 = x * x;
  return ((((70.0f * x - 315.0f) * x + 540.0f) * x - 420.0f) * x + 126.0f) * x2 * x2 * x;
}
// ---- src/math.rs:74-76 exp10, :289-291 db_amp
inline double exp10d(double x) { return exp(x * 2.302585092994046 /* LN_10 */); }
inline double db_ampd(double db) { return exp10d(db / 20.0); }

// ---- `wide 1.1.1` f32x8::round = round-half-even (roundps); src/lib.rs:326-328 F32x::floor.
inline float wide_roundf(float x) { return nearbyintf(x); }
inline float wide_floorf(float x) { return wide_roundf(x - 0.4999999f); }

// ---- `wide 1.1.1` f32x8::sin (call site src/oscillator.rs:82). Restated from the published
// algorithm (Agner Fog VCL `sincos_f`, Cephes single-precision coefficients); no FMA contraction
// (x86-64 baseline build has no `fma` target feature). Lane-wise scalar form.
inline float wide_sinf(float v) {
  const float DP1F = 0.78515625f * 2.0f;
  const float DP2F = 2.4187564849853515625E-4f * 2.0f;
  const float DP3F = 3.77489497744594108E-8f * 2.0f;
  const float P0SINF = -1.6666654611E-1f, P1SINF = 8.3321608736E-3f, P2SINF = -1.9515295891E-4f;
  const float P0COSF = 4.166664568298827E-2f, P1COSF = -1.388731625493765E-3f,
              P2COSF = 2.443315711809948E-5f;
  const float TWO_OVER_PI = 2.0f / 3.14159274101257324f;
  float xa = fabsf(v);
  float y = wide_roundf(xa * TWO_OVER_PI);
  // cvttps2dq: truncation in range, 0x80000000 for NaN and |y| >= 2^31 (finite |v| >~ 3.4e9); a plain cast would be undefined there
  int32_t q = (y >= -2147483648.0f && y < 2147483648.0f) ? (int32_t)y : INT32_MIN;
  float x = ((xa - y * DP1F) - y * DP2F) - y * DP3F;
  float x2 = x * x;
  float x4 = x2 * x2;
  float s = (x4 * P2SINF + (x2 * P1SINF + P0SINF)) * (x * x2) + x;
  float c = (x4 * P2COSF + (x2 * P1COSF + P0COSF)) * x4 + (1.0f - 0.5f * x2);
  if (q > 0x2000000 && std::isfinite(xa)) { s = 0.0f; c = 1.0f; }
  float r = (q & 1) ? c : s;
  uint32_t vb, rb;
  memcpy(&vb, &v, 4);
  memcpy(&rb, &r, 4);
  uint32_t sign = (((uint32_t)q << 30) ^ vb) & 0x80000000u;
  rb ^= sign;
  memcpy(&r, &rb, 4);
  return r;
}

}  // namespace fo

// fundsp_b200 device math substrate (sm_90a). Hand-written for the voice-bank kernels.
//
// Numeric contract (DESIGN.md §"Arithmetic"): every f32 operation is an individually rounded IEEE
// operation in the order the reference writes it (the reference is Rust: no a*b+c contraction), so this
// translation unit MUST be compiled with -fmad=false, without --use_fast_math, -ftz=false, -prec-div=true.
// Reference call sites are cited per function (paths relative to the reference checkout).
#pragma once

#ifdef __CUDACC_RTC__
typedef unsigned int uint32_t;
typedef int int32_t;
typedef unsigned long long uint64_t;
typedef long long int64_t;
#elif defined(FDSP_HOST_EMUL)
// tests/cpp/device_emul.cpp compiles this node library for the host CPU (TEST INFRASTRUCTURE: lets the CPU-only test suite run
// the device templates against the oracle; the product never defines FDSP_HOST_EMUL). Shims for the few intrinsics used.
#include <cmath>
#include <cstdint>
#include <cstring>
#define __device__
#define __host__
#define __forceinline__ inline
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
static inline float __fadd_rz(float a, float b) {   // exact when the f64 sum is (every use here: |a| < 2^23, b = 2^23)
  const double s = (double)a + (double)b;
  float f = (float)s;
  if (fabs((double)f) > fabs(s)) f = nextafterf(f, 0.0f);
  return f;
}
static inline int __popc(uint32_t x) { return __builtin_popcount(x); }
static inline double __longlong_as_double(long long x) { double d; memcpy(&d, &x, 8); return d; }
static inline long long __double_as_longlong(double d) { long long x; memcpy(&x, &d, 8); return x; }
using std::isfinite;
#else
#include <cstdint>
#include <cuda_runtime.h>
#endif

namespace fdsp {

#define FDSP_DEV __device__ __forceinline__
// cold paths that must NOT be inlined into a sample loop (coefficient recomputation behind an "input changed" test): one copy, out of line
#ifdef FDSP_HOST_EMUL
#define FDSP_COLD static inline
#else
#define FDSP_COLD static __device__ __noinline__
#endif

constexpr float TAU_F = 6.28318530717958647692f;  // f32::TAU
constexpr float PI_F = 3.14159265358979323846f;   // f32::PI

// reference src/noise.rs:150-157 hash32x
FDSP_DEV uint32_t hash32x(uint32_t x) {
  const uint32_t M = 0x45d9f3bu;
  x = (x ^ (x >> 16)) * M;
  x = (x ^ (x >> 16)) * M;
  return (x ^ (x >> 16)) * M;
}

// reference src/math.rs:569-576 rnd1 (used on device only by the envelope segment jitter, src/envelope.rs:249-253)
FDSP_DEV double rnd1(uint64_t x) {
  x ^= 0x5555555555555555ull;
  x *= 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  x = x ^ (x >> 31);
  return (double)(x >> 11) * (1.0 / 9007199254740992.0);
}

FDSP_DEV float lerpf(float a, float b, float t) { return a * (1.0f - t) + b * t; }   // src/math.rs:170-177
FDSP_DEV float delerpf(float a, float b, float x) { return (x - a) / (b - a); }      // src/math.rs:216-218
FDSP_DEV float clamp01f(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }             // src/math.rs:135-137
FDSP_DEV float clamp11f(float x) { return fminf(fmaxf(x, -1.0f), 1.0f); }            // src/math.rs:141-143

// `wide` f32x8::round (round half to even) and the reference's F32x::floor = (x - 0.4999999).round() (src/lib.rs:326-328)
FDSP_DEV float wide_roundf(float x) { return rintf(x); }
FDSP_DEV float wide_floorf(float x) { return rintf(x - 0.4999999f); }

// f32 -> i32 with the semantics of x86's cvttss2si / cvttps2dq, which `wide` and the host run: truncation toward zero in range, and
// INT32_MIN (0x80000000) for NaN and for |y| >= 2^31. A plain (int) cast is undefined there; PTX's cvt.rzi.s32.f32 saturates to
// 0x7fffffff and gives 0 for NaN.
FDSP_DEV int32_t cvtt_i32(float y) { return (y >= -2147483648.0f && y < 2147483648.0f) ? (int32_t)y : (int32_t)0x80000000u; }

// `wide` f32x8::sin as called by the block path of Sine (src/oscillator.rs:82): Cephes/VCL sincos, lane-wise.
FDSP_DEV float wide_sinf(float v) {
  const float DP1F = 0.78515625f * 2.0f;
  const float DP2F = 2.4187564849853515625E-4f * 2.0f;
  const float DP3F = 3.77489497744594108E-8f * 2.0f;
  const float P0SINF = -1.6666654611E-1f, P1SINF = 8.3321608736E-3f, P2SINF = -1.9515295891E-4f;
  const float P0COSF = 4.166664568298827E-2f, P1COSF = -1.388731625493765E-3f, P2COSF = 2.443315711809948E-5f;
  const float TWO_OVER_PI = 2.0f / 3.14159274101257324f;
  float xa = fabsf(v);
  float y = rintf(xa * TWO_OVER_PI);
  int q = cvtt_i32(y);
  float x = ((xa - y * DP1F) - y * DP2F) - y * DP3F;
  float x2 = x * x;
  float x4 = x2 * x2;
  float s = (x4 * P2SINF + (x2 * P1SINF + P0SINF)) * (x * x2) + x;
  float c = (x4 * P2COSF + (x2 * P1COSF + P0COSF)) * x4 + (1.0f - 0.5f * x2);
  if (q > 0x2000000 && isfinite(xa)) { s = 0.0f; c = 1.0f; }
  float r = (q & 1) ? c : s;
  uint32_t sign = (((uint32_t)q << 30) ^ __float_as_uint(v)) & 0x80000000u;
  return __uint_as_float(__float_as_uint(r) ^ sign);
}

// `wide` f32x8::atan as called by the block path of Shaper<Atan> (src/shape.rs:101-103): Cephes/VCL atan_f, lane-wise. Three ranges
// of t = |v| give z = t (t < sqrt2 - 1, offset 0), (t - 1) / (t + 1) (offset pi/4) or -1 / t (t > sqrt2 + 1, offset pi/2); a NaN falls
// in none of them and comes out of 0 / 0. polynomial_3 and mul_add without FMA, as wide_sinf; the sign is copied from v's sign bit.
FDSP_DEV float wide_atanf(float v) {
  const float P3 = 8.05374449538E-2f, P2 = -1.38776856032E-1f, P1 = 1.99777106478E-1f, P0 = -3.33329491539E-1f;
  const float SQRT_2 = 1.41421356237309504880f, FRAC_PI_4 = 0.785398163397448309616f, FRAC_PI_2 = 1.57079632679489661923f;
  const float t = fabsf(v);
  const bool notsmal = t >= SQRT_2 - 1.0f, notbig = t <= SQRT_2 + 1.0f;
  const float s = notsmal ? (notbig ? FRAC_PI_4 : FRAC_PI_2) : 0.0f;
  float a = notbig ? t : 0.0f;
  a = notsmal ? a - 1.0f : a;
  float b = notbig ? 1.0f : 0.0f;
  b = notsmal ? b + t : b;
  const float z = a / b;
  const float zz = z * z;
  const float x2 = zz * zz;
  float re = x2 * (P3 * zz + P2) + (P1 * zz + P0);
  re = (re * (zz * z) + z) + s;
  return (__float_as_uint(v) >> 31) ? -re : re;
}

// reference src/wavetable.rs:24-38 optimal4x44 (T = f32; f64 literals are rounded to f32 first)
FDSP_DEV float optimal4x44(float a0, float a1, float a2, float a3, float x) {
  float z = x - 0.5f;
  float even1 = a2 + a1, odd1 = a2 - a1, even2 = a3 + a0, odd2 = a3 - a0;
  float c0 = even1 * (float)0.4656725512077848 + even2 * (float)0.03432729708429672;
  float c1 = odd1 * (float)0.5374383075356016 + odd2 * (float)0.1542946255730746;
  float c2 = even1 * (float)-0.25194210134021744 + even2 * (float)0.2519474493593906;
  float c3 = odd1 * (float)-0.46896069955075126 + odd2 * (float)0.15578800670302476;
  float c4 = even1 * (float)0.00986988334359864 + even2 * (float)-0.00989340017126506;
  return (((c4 * z + c3) * z + c2) * z + c1) * z + c0;
}


// ---- 8-lane forms of the two functions above: identical per-lane operation order, written lane-parallel so that the
// eight independent evaluations overlap in one thread (the GPU counterpart of the reference's f32x8 arithmetic).
#define FDSP_L8 _Pragma("unroll") for (int j = 0; j < 8; j++)
FDSP_DEV void optimal4x44_8(const float* a0, const float* a1, const float* a2, const float* a3, const float* x, float* y) {
  float z[8], e1[8], o1[8], e2[8], o2[8], c0[8], c1[8], c2[8], c3[8], c4[8];
  FDSP_L8 z[j] = x[j] - 0.5f;
  FDSP_L8 { e1[j] = a2[j] + a1[j]; o1[j] = a2[j] - a1[j]; e2[j] = a3[j] + a0[j]; o2[j] = a3[j] - a0[j]; }
  FDSP_L8 c4[j] = e1[j] * (float)0.00986988334359864 + e2[j] * (float)-0.00989340017126506;
  FDSP_L8 c3[j] = o1[j] * (float)-0.46896069955075126 + o2[j] * (float)0.15578800670302476;
  FDSP_L8 c2[j] = e1[j] * (float)-0.25194210134021744 + e2[j] * (float)0.2519474493593906;
  FDSP_L8 c1[j] = o1[j] * (float)0.5374383075356016 + o2[j] * (float)0.1542946255730746;
  FDSP_L8 c0[j] = e1[j] * (float)0.4656725512077848 + e2[j] * (float)0.03432729708429672;
  FDSP_L8 y[j] = c4[j] * z[j] + c3[j];
  FDSP_L8 y[j] = y[j] * z[j] + c2[j];
  FDSP_L8 y[j] = y[j] * z[j] + c1[j];
  FDSP_L8 y[j] = y[j] * z[j] + c0[j];
}
FDSP_DEV void wide_sinf8(const float* v, float* out) {
  FDSP_L8 out[j] = wide_sinf(v[j]);
}
FDSP_DEV void wide_atanf8(const float* v, float* out) {
  FDSP_L8 out[j] = wide_atanf(v[j]);
}

}  // namespace fdsp

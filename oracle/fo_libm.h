// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h).
// Restatement of the scalar f32 libm functions the reference calls through the Rust `libm 0.2.15` crate
// (src/lib.rs:168-223,444-518,773-798: f32::sin/cos/tan -> libm::sinf/cosf/tanf, f32::tanh -> libm::tanhf).
// That crate is a port of musl libc's math library (FreeBSD msun lineage); its source is not in
// the reference crate, so the published algorithms are restated here:
//   sinf/cosf/tanf : k_sinf.c / k_cosf.c / k_tanf.c double-precision kernels + rem_pio2f "medium" reduction
//   expm1f, tanhf  : s_expm1f.c / s_tanhf.c
// PARITY UNPINNED at the ulp level against the real crate (no Rust toolchain here); tests pin these against
// glibc to <= 1 ulp over dense sweeps (tests/test_oracle.py::test_restated_libm_*), which would expose any
// mis-remembered constant. |x| >= 2^28*pi/2 takes rem_pio2f's large path (k_rem_pio2.c, Payne-Hanek), restated below: no f32 path
// calls the platform's sin/cos/tan.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace fo {
namespace m {

inline uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
inline float fromb(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }

// k_sinf.c
inline float k_sindf(double x) {
  const double S1 = -0x15555554cbac77.0p-55, S2 = 0x111110896efbb2.0p-59, S3 = -0x1a00f9e2cae774.0p-65, S4 = 0x16cd878c3b46a7.0p-71;
  double z = x * x;
  double w = z * z;
  double r = S3 + z * S4;
  double s = z * x;
  return (float)((x + s * (S1 + z * S2)) + s * w * r);
}
// k_cosf.c
inline float k_cosdf(double x) {
  const double C0 = -0x1ffffffd0c5e81.0p-54, C1 = 0x155553e1053a42.0p-57, C2 = -0x16c087e80f1e27.0p-62, C3 = 0x199342e0ee5069.0p-68;
  double z = x * x;
  double w = z * z;
  double r = C2 + z * C3;
  return (float)(((1.0 + z * C0) + w * C1) + (w * z) * r);
}
// k_tanf.c
inline float k_tandf(double x, int odd) {
  const double T0 = 0x15554d3418c99f.0p-54, T1 = 0x1112fd38999f72.0p-55, T2 = 0x1b54c91d865afe.0p-57, T3 = 0x191df3908c33ce.0p-58,
               T4 = 0x185dadfcecf44e.0p-61, T5 = 0x1362b9bf971bcd.0p-59;
  double z = x * x;
  double r = T4 + z * T5;
  double t = T2 + z * T3;
  double w = z * z;
  double s = z * x;
  double u = T0 + z * T1;
  r = (x + s * u) + (s * w) * (t + w * r);
  return (float)(odd ? -1.0 / r : r);
}
// rem_pio2f.c, medium-size path (|x| < 2^28 * pi/2)
inline int rem_pio2f_medium(float x, double* y) {
  const double TOINT = 1.5 / 2.220446049250313e-16, INV_PIO2 = 6.36619772367581382433e-01, PIO2_1 = 1.57079631090164184570e+00,
               PIO2_1T = 1.58932547735281966916e-08;
  double x64 = (double)x;
  double tmp = x64 * INV_PIO2 + TOINT;
  double fn = tmp - TOINT;
  *y = x64 - fn * PIO2_1 - fn * PIO2_1T;
  return (int)(int32_t)fn;
}
// k_rem_pio2.c __rem_pio2_large(x, y, e0, nx, prec) for prec 0 (one double out), as rem_pio2f.c calls it with nx = 1.
static const int32_t IPIO2[] = {   // 2/pi in 24-bit digits
  0xA2F983, 0x6E4E44, 0x1529FC, 0x2757D1, 0xF534DD, 0xC0DB62, 0x95993C, 0x439041, 0xFE5163, 0xABDEBB, 0xC561B7, 0x246E3A,
  0x424DD2, 0xE00649, 0x2EEA09, 0xD1921C, 0xFE1DEB, 0x1CB129, 0xA73EE8, 0x8235F5, 0x2EBB44, 0x84E99C, 0x7026B4, 0x5F7E41,
  0x3991D6, 0x398353, 0x39F49C, 0x845F8B, 0xBDF928, 0x3B1FF8, 0x97FFDE, 0x05980F};
static const double PIO2_PIECES[] = {1.57079625129699707031e+00, 7.54978941586159635335e-08, 5.39030252995776476554e-15,
                                     3.28200341580791294123e-22, 1.27065575308067607349e-29, 1.22933308981111328932e-36,
                                     2.73370053816464559624e-44, 2.16741683877804819444e-51};
inline double scalbn_exact(double x, int n) {   // x * 2^n for the small |n| used here (never leaves the normal range)
  uint64_t u = (uint64_t)(0x3ff + n) << 52; double p; memcpy(&p, &u, 8); return x * p;
}
inline int rem_pio2_large(const double* x, double* y, int e0, int nx) {
  const int jk = 3, jp = jk;   // init_jk[prec = 0]
  int32_t jz, jx, jv, carry, n, iq[20], i, j, k, m, q0, ih;
  double z, fw, f[20], fq[20], q[20];
  jx = nx - 1;
  jv = (e0 - 3) / 24; if (jv < 0) jv = 0;
  q0 = e0 - 24 * (jv + 1);
  j = jv - jx; m = jx + jk;
  for (i = 0; i <= m; i++, j++) f[i] = j < 0 ? 0.0 : (double)IPIO2[j];
  for (i = 0; i <= jk; i++) { for (j = 0, fw = 0.0; j <= jx; j++) fw += x[j] * f[jx + i - j]; q[i] = fw; }
  jz = jk;
recompute:
  for (i = 0, j = jz, z = q[jz]; j > 0; i++, j--) {
    fw = (double)(int32_t)(0x1p-24 * z);
    iq[i] = (int32_t)(z - 0x1p24 * fw);
    z = q[j - 1] + fw;
  }
  z = scalbn_exact(z, q0);
  z -= 8.0 * std::floor(z * 0.125);
  n = (int32_t)z;
  z -= (double)n;
  ih = 0;
  if (q0 > 0) {
    i = iq[jz - 1] >> (24 - q0); n += i;
    iq[jz - 1] -= i << (24 - q0);
    ih = iq[jz - 1] >> (23 - q0);
  } else if (q0 == 0) ih = iq[jz - 1] >> 23;
  else if (z >= 0.5) ih = 2;
  if (ih > 0) {
    n += 1; carry = 0;
    for (i = 0; i < jz; i++) {
      j = iq[i];
      if (carry == 0) {
        if (j != 0) { carry = 1; iq[i] = 0x1000000 - j; }
      } else iq[i] = 0xffffff - j;
    }
    if (q0 > 0) {
      switch (q0) { case 1: iq[jz - 1] &= 0x7fffff; break; case 2: iq[jz - 1] &= 0x3fffff; break; }
    }
    if (ih == 2) { z = 1.0 - z; if (carry != 0) z -= scalbn_exact(1.0, q0); }
  }
  if (z == 0) {
    j = 0;
    for (i = jz - 1; i >= jk; i--) j |= iq[i];
    if (j == 0) {
      for (k = 1; iq[jk - k] == 0; k++) {}
      for (i = jz + 1; i <= jz + k; i++) {
        f[jx + i] = (double)IPIO2[jv + i];
        for (j = 0, fw = 0.0; j <= jx; j++) fw += x[j] * f[jx + i - j];
        q[i] = fw;
      }
      jz += k;
      goto recompute;
    }
  }
  if (z == 0.0) {
    jz -= 1; q0 -= 24;
    while (iq[jz] == 0) { jz--; q0 -= 24; }
  } else {
    z = scalbn_exact(z, -q0);
    if (z >= 0x1p24) {
      fw = (double)(int32_t)(0x1p-24 * z);
      iq[jz] = (int32_t)(z - 0x1p24 * fw);
      jz += 1; q0 += 24;
      iq[jz] = (int32_t)fw;
    } else iq[jz] = (int32_t)z;
  }
  fw = scalbn_exact(1.0, q0);
  for (i = jz; i >= 0; i--) { q[i] = fw * (double)iq[i]; fw *= 0x1p-24; }
  for (i = jz; i >= 0; i--) {
    for (fw = 0.0, k = 0; k <= jp && k <= jz - i; k++) fw += PIO2_PIECES[k] * q[i + k];
    fq[jz - i] = fw;
  }
  fw = 0.0;
  for (i = jz; i >= 0; i--) fw += fq[i];
  y[0] = ih == 0 ? fw : -fw;
  return n & 7;
}
// rem_pio2f.c: the medium path below 2^28 * pi/2, else x scaled into [2^23, 2^24) and handed to rem_pio2_large (x finite)
inline int rem_pio2f_(float x, double* y) {
  const uint32_t hx = fbits(x), ix = hx & 0x7fffffffu;
  if (ix < 0x4dc90fdbu) return rem_pio2f_medium(x, y);
  const int32_t e0 = (int32_t)(ix >> 23) - (0x7f + 23);
  double tx[1], ty[1];
  tx[0] = (double)fromb(ix - ((uint32_t)e0 << 23));
  const int n = rem_pio2_large(tx, ty, e0, 1);
  if (hx >> 31) { *y = -ty[0]; return -n; }
  *y = ty[0];
  return n;
}
const double S1PIO2 = 1.0 * 1.57079632679489661923, S2PIO2 = 2.0 * 1.57079632679489661923, S3PIO2 = 3.0 * 1.57079632679489661923,
             S4PIO2 = 4.0 * 1.57079632679489661923;

inline float sinf_(float x) {  // sinf.c
  uint32_t ix = fbits(x); int sign = (int)(ix >> 31); ix &= 0x7fffffffu;
  if (ix <= 0x3f490fdau) { if (ix < 0x39800000u) return x; return k_sindf((double)x); }
  if (ix <= 0x407b53d1u) {
    if (ix <= 0x4016cbe3u) return sign ? -k_cosdf((double)x + S1PIO2) : k_cosdf((double)x - S1PIO2);
    return k_sindf(sign ? -((double)x + S2PIO2) : -((double)x - S2PIO2));
  }
  if (ix <= 0x40e231d5u) {
    if (ix <= 0x40afeddfu) return sign ? k_cosdf((double)x + S3PIO2) : -k_cosdf((double)x - S3PIO2);
    return k_sindf(sign ? (double)x + S4PIO2 : (double)x - S4PIO2);
  }
  if (ix >= 0x7f800000u) return x - x;
  double y; int n = rem_pio2f_(x, &y);
  switch (n & 3) { case 0: return k_sindf(y); case 1: return k_cosdf(y); case 2: return k_sindf(-y); default: return -k_cosdf(y); }
}
inline float cosf_(float x) {  // cosf.c
  uint32_t ix = fbits(x); int sign = (int)(ix >> 31); ix &= 0x7fffffffu;
  if (ix <= 0x3f490fdau) { if (ix < 0x39800000u) return 1.0f; return k_cosdf((double)x); }
  if (ix <= 0x407b53d1u) {
    if (ix > 0x4016cbe3u) return -k_cosdf(sign ? (double)x + S2PIO2 : (double)x - S2PIO2);
    return sign ? k_sindf((double)x + S1PIO2) : k_sindf(S1PIO2 - (double)x);
  }
  if (ix <= 0x40e231d5u) {
    if (ix > 0x40afeddfu) return k_cosdf(sign ? (double)x + S4PIO2 : (double)x - S4PIO2);
    return sign ? k_sindf(-(double)x - S3PIO2) : k_sindf((double)x - S3PIO2);
  }
  if (ix >= 0x7f800000u) return x - x;
  double y; int n = rem_pio2f_(x, &y);
  switch (n & 3) { case 0: return k_cosdf(y); case 1: return k_sindf(-y); case 2: return -k_cosdf(y); default: return k_sindf(y); }
}
inline float tanf_(float x) {  // tanf.c
  uint32_t ix = fbits(x); int sign = (int)(ix >> 31); ix &= 0x7fffffffu;
  if (ix <= 0x3f490fdau) { if (ix < 0x39800000u) return x; return k_tandf((double)x, 0); }
  if (ix <= 0x407b53d1u) {
    if (ix <= 0x4016cbe3u) return k_tandf(sign ? (double)x + S1PIO2 : (double)x - S1PIO2, 1);
    return k_tandf(sign ? (double)x + S2PIO2 : (double)x - S2PIO2, 0);
  }
  if (ix <= 0x40e231d5u) {
    if (ix <= 0x40afeddfu) return k_tandf(sign ? (double)x + S3PIO2 : (double)x - S3PIO2, 1);
    return k_tandf(sign ? (double)x + S4PIO2 : (double)x - S4PIO2, 0);
  }
  if (ix >= 0x7f800000u) return x - x;
  double y; int n = rem_pio2f_(x, &y);
  return k_tandf(y, n & 1);
}

inline float expm1f_(float x) {  // s_expm1f.c
  const float ln2_hi = 6.9313812256e-01f, ln2_lo = 9.0580006145e-06f, invln2 = 1.4426950216e+00f, Q1 = -3.3333212137e-2f, Q2 = 1.5807170421e-3f;
  float y, hi, lo, c = 0.0f, t, e, hxs, hfx, r1, twopk;
  uint32_t hx = fbits(x) & 0x7fffffffu; int k, sign = (int)(fbits(x) >> 31);
  if (hx >= 0x4195b844u) {  // |x| >= 27 ln2
    if (hx > 0x7f800000u) return x;
    if (sign) return -1.0f;
    if (hx > 0x42b17217u) { x *= 0x1p127f; return x; }
  }
  if (hx > 0x3eb17218u) {  // |x| > 0.5 ln2
    if (hx < 0x3F851592u) {  // |x| < 1.5 ln2
      if (!sign) { hi = x - ln2_hi; lo = ln2_lo; k = 1; } else { hi = x + ln2_hi; lo = -ln2_lo; k = -1; }
    } else {
      k = (int)(invln2 * x + (sign ? -0.5f : 0.5f));
      t = (float)k;
      hi = x - t * ln2_hi;
      lo = t * ln2_lo;
    }
    x = hi - lo;
    c = (hi - x) - lo;
  } else if (hx < 0x33000000u) {
    return x;
  } else k = 0;
  hfx = 0.5f * x;
  hxs = x * hfx;
  r1 = 1.0f + hxs * (Q1 + hxs * Q2);
  t = 3.0f - r1 * hfx;
  e = hxs * ((r1 - t) / (6.0f - x * t));
  if (k == 0) return x - (x * e - hxs);
  e = x * (e - c) - c;
  e -= hxs;
  if (k == -1) return 0.5f * (x - e) - 0.5f;
  if (k == 1) { if (x < -0.25f) return -2.0f * (e - (x + 0.5f)); return 1.0f + 2.0f * (x - e); }
  twopk = fromb((uint32_t)(0x7f + k) << 23);
  if (k < 0 || k > 56) {
    y = x - e + 1.0f;
    if (k == 128) y = y * 2.0f * 0x1p127f; else y = y * twopk;
    return y - 1.0f;
  }
  float uf = fromb((uint32_t)(0x7f - k) << 23);
  if (k < 23) y = (x - e + (1.0f - uf)) * twopk; else y = (x - (e + uf) + 1.0f) * twopk;
  return y;
}

// e_expf.c (FreeBSD msun lineage, as ported by the Rust `libm` crate) + s_scalbnf.c
inline float scalbnf_(float x, int n) {
  float y = x;
  if (n > 127) { y *= 0x1p127f; n -= 127; if (n > 127) { y *= 0x1p127f; n -= 127; if (n > 127) n = 127; } }
  else if (n < -126) { y *= 0x1p-126f * 0x1p24f; n += 126 - 24; if (n < -126) { y *= 0x1p-126f * 0x1p24f; n += 126 - 24; if (n < -126) n = -126; } }
  return y * fromb((uint32_t)(0x7f + n) << 23);
}
inline float expf_(float x) {
  const float LN2_HI = 6.9314575195e-01f, LN2_LO = 1.4286067653e-06f, INV_LN2 = 1.4426950216e+00f, P1 = 1.6666625440e-1f, P2 = -2.7667332906e-3f;
  uint32_t hx = fbits(x); const int sign = (int)(hx >> 31); hx &= 0x7fffffffu;
  if (hx >= 0x42aeac50u) {                 // |x| >= 87.33655 or NaN
    if (hx > 0x7f800000u) return x;
    if (hx >= 0x42b17218u && !sign) { x *= 0x1p127f; return x; }
    if (sign && hx >= 0x42cff1b5u) return 0.0f;
  }
  int k; float hi, lo;
  if (hx > 0x3eb17218u) {                  // |x| > 0.5 ln2
    if (hx > 0x3f851592u) k = (int)(INV_LN2 * x + (sign ? -0.5f : 0.5f)); else k = 1 - sign - sign;
    const float kf = (float)k;
    hi = x - kf * LN2_HI; lo = kf * LN2_LO; x = hi - lo;
  } else if (hx > 0x39000000u) { k = 0; hi = x; lo = 0.0f; }
  else return 1.0f + x;
  const float xx = x * x;
  const float c = x - xx * (P1 + xx * P2);
  const float y = 1.0f + (x * c / (2.0f - c) - lo + hi);
  return k == 0 ? y : scalbnf_(y, k);
}
// e_powf.c (FreeBSD msun lineage, as ported by the Rust `libm` crate, src/math/powf.rs): float-only arithmetic,
// log2(x) in two pieces (t1 + t2), y*log2(x) split the same way, then 2**(p_h + p_l).
inline float powf_(float x, float y) {
  const float two24 = 16777216.0f, huge = 1.0e30f, tiny = 1.0e-30f;
  const float L1 = 6.0000002384e-01f, L2 = 4.2857143283e-01f, L3 = 3.3333334327e-01f, L4 = 2.7272811532e-01f, L5 = 2.3066075146e-01f, L6 = 2.0697501302e-01f;
  const float P1 = 1.6666667163e-01f, P2 = -2.7777778450e-03f, P3 = 6.6137559770e-05f, P4 = -1.6533901999e-06f, P5 = 4.1381369442e-08f;
  const float lg2 = 6.9314718246e-01f, lg2_h = 6.93145752e-01f, lg2_l = 1.42860654e-06f, ovt = 4.2995665694e-08f;
  const float cp = 9.6179670095e-01f, cp_h = 9.6191406250e-01f, cp_l = -1.1736857402e-04f;
  const float ivln2 = 1.4426950216e+00f, ivln2_h = 1.4426879883e+00f, ivln2_l = 7.0526075433e-06f;
  float z, ax, z_h, z_l, p_h, p_l, y1, t1, t2, r, s, sn, t, u, v, w;
  int32_t i, j, k, yisint, n, is;
  const int32_t hx = (int32_t)fbits(x), hy = (int32_t)fbits(y);
  int32_t ix = hx & 0x7fffffff;
  const int32_t iy = hy & 0x7fffffff;
  if (iy == 0) return 1.0f;                    // x**0 = 1, even if x is NaN
  if (hx == 0x3f800000) return 1.0f;           // 1**y = 1, even if y is NaN
  if (ix > 0x7f800000 || iy > 0x7f800000) return x + y;
  yisint = 0;                                   // 0: y not an integer, 1: odd, 2: even (only needed for x < 0)
  if (hx < 0) {
    if (iy >= 0x4b800000) yisint = 2;
    else if (iy >= 0x3f800000) {
      k = (iy >> 23) - 0x7f;
      j = iy >> (23 - k);
      if ((j << (23 - k)) == iy) yisint = 2 - (j & 1);
    }
  }
  if (iy == 0x7f800000) {                       // y is +-inf
    if (ix == 0x3f800000) return 1.0f;
    else if (ix > 0x3f800000) return hy >= 0 ? y : 0.0f;
    else return hy >= 0 ? 0.0f : -y;
  }
  if (iy == 0x3f800000) return hy >= 0 ? x : 1.0f / x;
  if (hy == 0x40000000) return x * x;
  if (hy == 0x3f000000 && hx >= 0) return sqrtf(x);
  ax = fromb((uint32_t)ix);
  if (ix == 0x7f800000 || ix == 0 || ix == 0x3f800000) {   // x is +-0, +-inf, +-1
    z = ax;
    if (hy < 0) z = 1.0f / z;
    if (hx < 0) {
      if (((ix - 0x3f800000) | yisint) == 0) z = (z - z) / (z - z);
      else if (yisint == 1) z = -z;
    }
    return z;
  }
  sn = 1.0f;
  if (hx < 0) {
    if (yisint == 0) return (x - x) / (x - x);
    if (yisint == 1) sn = -1.0f;
  }
  if (iy > 0x4d000000) {                        // |y| > 2**27
    if (ix < 0x3f7ffff8) return hy < 0 ? sn * huge * huge : sn * tiny * tiny;
    if (ix > 0x3f800007) return hy > 0 ? sn * huge * huge : sn * tiny * tiny;
    t = ax - 1.0f;
    w = (t * t) * (0.5f - t * (0.333333333333f - t * 0.25f));
    u = ivln2_h * t;
    v = t * ivln2_l - w * ivln2;
    t1 = u + v;
    t1 = fromb(fbits(t1) & 0xfffff000u);
    t2 = v - (t1 - u);
  } else {
    float s2, s_h, s_l, t_h, t_l;
    n = 0;
    if (ix < 0x00800000) { ax *= two24; n -= 24; ix = (int32_t)fbits(ax); }
    n += (ix >> 23) - 0x7f;
    j = ix & 0x007fffff;
    ix = j | 0x3f800000;
    if (j <= 0x1cc471) k = 0;                   // |x| < sqrt(3/2)
    else if (j < 0x5db3d7) k = 1;               // |x| < sqrt(3)
    else { k = 0; n += 1; ix -= 0x00800000; }
    ax = fromb((uint32_t)ix);
    const float bpk = k ? 1.5f : 1.0f, dp_hk = k ? 5.84960938e-01f : 0.0f, dp_lk = k ? 1.56322085e-06f : 0.0f;
    u = ax - bpk;
    v = 1.0f / (ax + bpk);
    s = u * v;
    s_h = fromb(fbits(s) & 0xfffff000u);
    is = (int32_t)((((uint32_t)ix >> 1) & 0xfffff000u) | 0x20000000u);
    t_h = fromb((uint32_t)(is + 0x00400000 + (k << 21)));
    t_l = ax - (t_h - bpk);
    s_l = v * ((u - s_h * t_h) - s_h * t_l);
    s2 = s * s;
    r = s2 * s2 * (L1 + s2 * (L2 + s2 * (L3 + s2 * (L4 + s2 * (L5 + s2 * L6)))));
    r += s_l * (s_h + s);
    s2 = s_h * s_h;
    t_h = 3.0f + s2 + r;
    t_h = fromb(fbits(t_h) & 0xfffff000u);
    t_l = r - ((t_h - 3.0f) - s2);
    u = s_h * t_h;
    v = s_l * t_h + t_l * s;
    p_h = u + v;
    p_h = fromb(fbits(p_h) & 0xfffff000u);
    p_l = v - (p_h - u);
    z_h = cp_h * p_h;
    z_l = cp_l * p_h + p_l * cp + dp_lk;
    t = (float)n;
    t1 = (((z_h + z_l) + dp_hk) + t);
    t1 = fromb(fbits(t1) & 0xfffff000u);
    t2 = z_l - (((t1 - t) - dp_hk) - z_h);
  }
  y1 = fromb(fbits(y) & 0xfffff000u);
  p_l = (y - y1) * t1 + y * t2;
  p_h = y1 * t1;
  z = p_l + p_h;
  j = (int32_t)fbits(z);
  if (j > 0x43000000) return sn * huge * huge;
  else if (j == 0x43000000) { if (p_l + ovt > z - p_h) return sn * huge * huge; }
  else if ((j & 0x7fffffff) > 0x43160000) return sn * tiny * tiny;
  else if ((uint32_t)j == 0xc3160000u) { if (p_l <= z - p_h) return sn * tiny * tiny; }
  i = j & 0x7fffffff;
  k = (i >> 23) - 0x7f;
  n = 0;
  if (i > 0x3f000000) {                         // |z| > 0.5: n = [z + 0.5]
    n = j + (0x00800000 >> (k + 1));
    k = ((n & 0x7fffffff) >> 23) - 0x7f;
    t = fromb((uint32_t)(n & ~(0x007fffff >> k)));
    n = ((n & 0x007fffff) | 0x00800000) >> (23 - k);
    if (j < 0) n = -n;
    p_h -= t;
  }
  t = p_l + p_h;
  t = fromb(fbits(t) & 0xffff8000u);
  u = t * lg2_h;
  v = (p_l - (t - p_h)) * lg2 + t * lg2_l;
  z = u + v;
  w = v - (z - u);
  t = z * z;
  t1 = z - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))));
  r = (z * t1) / (t1 - 2.0f) - (w + z * w);
  z = 1.0f - (r - z);
  j = (int32_t)fbits(z);
  j += (int32_t)((uint32_t)n << 23);
  if ((j >> 23) <= 0) z = scalbnf_(z, n); else z = fromb((uint32_t)j);
  return sn * z;
}
inline float tanhf_(float x) {  // s_tanhf.c
  uint32_t w = fbits(x); int sign = (int)(w >> 31); w &= 0x7fffffffu;
  x = fromb(w);
  float t;
  if (w > 0x3f0c9f54u) {        // |x| > log(3)/2 or nan
    if (w > 0x41200000u) t = 1.0f + 0.0f / x;
    else { t = expm1f_(2.0f * x); t = 1.0f - 2.0f / (t + 2.0f); }
  } else if (w > 0x3e82c578u) {  // |x| > log(5/3)/2
    t = expm1f_(2.0f * x); t = t / (t + 2.0f);
  } else if (w >= 0x00800000u) {
    t = expm1f_(-2.0f * x); t = -t / (t + 2.0f);
  } else t = x;
  return sign ? -t : t;
}

}  // namespace m
}  // namespace fo

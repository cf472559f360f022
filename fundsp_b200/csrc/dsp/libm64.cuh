// fundsp_b200 scalar f64 math: sin/cos/tan/exp as the Rust `libm` crate (0.2.15) ports them from musl / FreeBSD msun (k_sin.c, k_cos.c,
// k_tan.c, e_rem_pio2.c, s_sin.c, s_cos.c, s_tan.c, e_exp.c). This is what the reference's f64 nodes call for their coefficients
// (reference src/lib.rs:520-568: `Float for f64`). Host and device share this one implementation, so coefficients computed at lowering
// time and those recomputed per sample on the device agree bit for bit.
//
// Argument reduction: |x| < 2^20 * pi/2 is reduced with e_rem_pio2's Cody-Waite steps (three rounds at most, exact to 151 bits).
// Larger finite arguments (k_rem_pio2.c's Payne-Hanek path) are NOT restated: they go to the platform's sin/cos/tan (CUDA's on the
// device, the C library's on the host), which may differ from msun in the last bit and between host and device. No node reaches
// them: the filters evaluate tan(pi * f / sr) and cos(tau * f / sr) for audible f.
#pragma once
#include "libm.cuh"

namespace fdsp {
namespace m64 {

FDSP_HD uint64_t dbits(double x) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__double_as_longlong(x);
#else
  uint64_t u; memcpy(&u, &x, 8); return u;
#endif
}
FDSP_HD double dfromb(uint64_t u) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)u);
#else
  double x; memcpy(&x, &u, 8); return x;
#endif
}
FDSP_HD uint32_t hiword(double x) { return (uint32_t)(dbits(x) >> 32); }
FDSP_HD double zero_low_word(double x) { return dfromb(dbits(x) & 0xffffffff00000000ull); }

// k_sin.c: sin(x + y) for |x| <= pi/4, y the tail of x (iy = 0: y is zero)
FDSP_HD double k_sin(double x, double y, int iy) {
  const double S1 = dfromb(0xBFC5555555555549ull), S2 = dfromb(0x3F8111111110F8A6ull), S3 = dfromb(0xBF2A01A019C161D5ull),
               S4 = dfromb(0x3EC71DE357B1FE7Dull), S5 = dfromb(0xBE5AE5E68A2B9CEBull), S6 = dfromb(0x3DE5D93A5ACFD57Cull);
  const double z = x * x;
  const double w = z * z;
  const double r = S2 + z * (S3 + z * S4) + z * w * (S5 + z * S6);
  const double v = z * x;
  if (iy == 0) return x + v * (S1 + z * r);
  return x - ((z * (0.5 * y - v * r) - y) - v * S1);
}
// k_cos.c: cos(x + y) for |x| <= pi/4
FDSP_HD double k_cos(double x, double y) {
  const double C1 = dfromb(0x3FA555555555554Cull), C2 = dfromb(0xBF56C16C16C15177ull), C3 = dfromb(0x3EFA01A019CB1590ull),
               C4 = dfromb(0xBE927E4F809C52ADull), C5 = dfromb(0x3E21EE9EBDB4B1C4ull), C6 = dfromb(0xBDA8FAE9BE8838D4ull);
  const double z = x * x;
  double w = z * z;
  const double r = z * (C1 + z * (C2 + z * C3)) + w * w * (C4 + z * (C5 + z * C6));
  const double hz = 0.5 * z;
  w = 1.0 - hz;
  return w + (((1.0 - w) - hz) + (z * r - x * y));
}
// k_tan.c (musl form): tan(x + y) (odd = 0) or -1 / tan(x + y) (odd = 1) for |x| <= pi/4
FDSP_HD double k_tan(double x, double y, int odd) {
  const double T[13] = {dfromb(0x3FD5555555555563ull), dfromb(0x3FC111111110FE7Aull), dfromb(0x3FABA1BA1BB341FEull), dfromb(0x3F9664F48406D637ull),
                        dfromb(0x3F8226E3E96E8493ull), dfromb(0x3F6D6D22C9560328ull), dfromb(0x3F57DBC8FEE08315ull), dfromb(0x3F4344D8F2F26501ull),
                        dfromb(0x3F3026F71A8D1068ull), dfromb(0x3F147E88A03792A6ull), dfromb(0x3F12B80F32F0A7E9ull), dfromb(0xBEF375CBDB605373ull),
                        dfromb(0x3EFB2A7074BF7AD4ull)};
  const double PIO4 = dfromb(0x3FE921FB54442D18ull), PIO4_LO = dfromb(0x3C81A62633145C07ull);
  const uint32_t hx = hiword(x);
  const bool big = (hx & 0x7fffffffu) >= 0x3FE59428u;   // |x| >= 0.6744
  if (big) {
    if (hx >> 31) { x = -x; y = -y; }
    x = (PIO4 - x) + (PIO4_LO - y);
    y = 0.0;
  }
  const double z = x * x;
  const double w = z * z;
  const double r0 = T[1] + w * (T[3] + w * (T[5] + w * (T[7] + w * (T[9] + w * T[11]))));
  const double v0 = z * (T[2] + w * (T[4] + w * (T[6] + w * (T[8] + w * (T[10] + w * T[12])))));
  const double s = z * x;
  const double r = y + z * (s * (r0 + v0) + y) + s * T[0];
  const double ww = x + r;
  if (big) {
    const double sg = 1.0 - 2.0 * (double)odd;
    const double v = sg - 2.0 * (x + (r - ww * ww / (ww + sg)));
    return (hx >> 31) ? -v : v;
  }
  if (odd == 0) return ww;
  const double w0 = zero_low_word(ww);   // -1 / (x + r) to within an ulp: a0 + a (1 + a0 w0 + a0 v) with w0 + v = x + r
  const double v = r - (w0 - x);
  const double a = -1.0 / ww;
  const double a0 = zero_low_word(a);
  return a0 + a * (1.0 + a0 * w0 + a0 * v);
}

// e_rem_pio2.c: x = n pi/2 + (y0 + y1), |y0 + y1| <= pi/4, for finite |x| < 2^20 pi/2 (the caller handles larger and non-finite x)
struct Rem { int n; double y0, y1; };
FDSP_HD Rem rem_pio2_medium(double x, uint32_t ix) {
  const double TOINT = 6755399441055744.0;   // 1.5 / EPSILON
  const double INV_PIO2 = dfromb(0x3FE45F306DC9C883ull);
  const double PIO2_1 = dfromb(0x3FF921FB54400000ull), PIO2_1T = dfromb(0x3DD0B4611A626331ull);
  const double PIO2_2 = dfromb(0x3DD0B4611A600000ull), PIO2_2T = dfromb(0x3BA3198A2E037073ull);
  const double PIO2_3 = dfromb(0x3BA3198A2E000000ull), PIO2_3T = dfromb(0x397B839A252049C1ull);
  const double tmp = x * INV_PIO2 + TOINT;
  const double fn = tmp - TOINT;
  const int n = (int)fn;
  double r = x - fn * PIO2_1;
  double w = fn * PIO2_1T;                   // first round, good to 85 bits
  double y0 = r - w;
  const int ex = (int)(ix >> 20);
  if (ex - (int)((dbits(y0) >> 52) & 0x7ff) > 16) {
    double t = r;                            // second round, good to 118 bits
    w = fn * PIO2_2;
    r = t - w;
    w = fn * PIO2_2T - ((t - r) - w);
    y0 = r - w;
    if (ex - (int)((dbits(y0) >> 52) & 0x7ff) > 49) {
      t = r;                                 // third round, good to 151 bits
      w = fn * PIO2_3;
      r = t - w;
      w = fn * PIO2_3T - ((t - r) - w);
      y0 = r - w;
    }
  }
  Rem q; q.n = n; q.y0 = y0; q.y1 = (r - y0) - w;
  return q;
}
FDSP_HD Rem rem_pio2_k(double x, int k, bool neg) {   // |x| near k pi/2, k = 1..4: one round with k * (pio2_1 + pio2_1t)
  const double P1 = (double)k * dfromb(0x3FF921FB54400000ull), P1T = (double)k * dfromb(0x3DD0B4611A626331ull);
  Rem q;
  if (!neg) { const double z = x - P1; q.y0 = z - P1T; q.y1 = (z - q.y0) - P1T; q.n = k; }
  else { const double z = x + P1; q.y0 = z + P1T; q.y1 = (z - q.y0) + P1T; q.n = -k; }
  return q;
}
// true when x is reduced here; false for |x| >= 2^20 pi/2 (the large-argument path this file does not restate)
FDSP_HD bool rem_pio2(double x, Rem& q) {
  const uint32_t ix = hiword(x) & 0x7fffffffu;
  const bool neg = (dbits(x) >> 63) != 0;
  if (ix <= 0x400f6a7au) {                                   // |x| ~<= 5pi/4
    if ((ix & 0xfffffu) == 0x921fbu) { q = rem_pio2_medium(x, ix); return true; }   // |x| ~= pi/2 or pi: cancellation
    q = rem_pio2_k(x, ix <= 0x4002d97cu ? 1 : 2, neg);       // 3pi/4 splits the two
    return true;
  }
  if (ix <= 0x401c463bu) {                                   // |x| ~<= 9pi/4
    if (ix <= 0x4015fdbcu) {                                 // |x| ~<= 7pi/4
      if (ix == 0x4012d97cu) { q = rem_pio2_medium(x, ix); return true; }            // |x| ~= 3pi/2
      q = rem_pio2_k(x, 3, neg);
    } else {
      if (ix == 0x401921fbu) { q = rem_pio2_medium(x, ix); return true; }            // |x| ~= 2pi
      q = rem_pio2_k(x, 4, neg);
    }
    return true;
  }
  if (ix < 0x413921fbu) { q = rem_pio2_medium(x, ix); return true; }                  // |x| ~< 2^20 pi/2
  return false;
}

FDSP_HD double sin(double x) {   // s_sin.c
  const uint32_t ix = hiword(x) & 0x7fffffffu;
  if (ix <= 0x3fe921fbu) {                                   // |x| ~<= pi/4
    if (ix < 0x3e500000u) return x;                          // |x| < 2^-26
    return k_sin(x, 0.0, 0);
  }
  if (ix >= 0x7ff00000u) return x - x;                       // inf or NaN
  Rem q;
  if (!rem_pio2(x, q)) return ::sin(x);
  switch (q.n & 3) {
    case 0: return k_sin(q.y0, q.y1, 1);
    case 1: return k_cos(q.y0, q.y1);
    case 2: return -k_sin(q.y0, q.y1, 1);
    default: return -k_cos(q.y0, q.y1);
  }
}
FDSP_HD double cos(double x) {   // s_cos.c
  const uint32_t ix = hiword(x) & 0x7fffffffu;
  if (ix <= 0x3fe921fbu) {
    if (ix < 0x3e46a09eu) return 1.0;                        // |x| < 2^-27 sqrt(2)
    return k_cos(x, 0.0);
  }
  if (ix >= 0x7ff00000u) return x - x;
  Rem q;
  if (!rem_pio2(x, q)) return ::cos(x);
  switch (q.n & 3) {
    case 0: return k_cos(q.y0, q.y1);
    case 1: return -k_sin(q.y0, q.y1, 1);
    case 2: return -k_cos(q.y0, q.y1);
    default: return k_sin(q.y0, q.y1, 1);
  }
}
FDSP_HD double tan(double x) {   // s_tan.c
  const uint32_t ix = hiword(x) & 0x7fffffffu;
  if (ix <= 0x3fe921fbu) {
    if (ix < 0x3e400000u) return x;                          // |x| < 2^-27
    return k_tan(x, 0.0, 0);
  }
  if (ix >= 0x7ff00000u) return x - x;
  Rem q;
  if (!rem_pio2(x, q)) return ::tan(x);
  return k_tan(q.y0, q.y1, q.n & 1);
}

// scalbn: y * 2^n, correctly rounded (musl's three-step form, which never rounds twice in the subnormal range)
FDSP_HD double scalbn(double y, int n) {
  const double X1P1023 = dfromb(0x7fe0000000000000ull), X1P_1022_53 = dfromb(0x0010000000000000ull) * dfromb(0x4340000000000000ull);
  if (n > 1023) {
    y *= X1P1023; n -= 1023;
    if (n > 1023) { y *= X1P1023; n -= 1023; if (n > 1023) n = 1023; }
  } else if (n < -1022) {
    y *= X1P_1022_53; n += 1022 - 53;
    if (n < -1022) { y *= X1P_1022_53; n += 1022 - 53; if (n < -1022) n = -1022; }
  }
  return y * dfromb((uint64_t)(0x3ff + n) << 52);
}
FDSP_HD double exp(double x) {   // e_exp.c
  const double LN2HI = dfromb(0x3FE62E42FEE00000ull), LN2LO = dfromb(0x3DEA39EF35793C76ull), INVLN2 = dfromb(0x3FF71547652B82FEull);
  const double P1 = dfromb(0x3FC555555555553Eull), P2 = dfromb(0xBF66C16C16BEBD93ull), P3 = dfromb(0x3F11566AAF25DE2Cull),
               P4 = dfromb(0xBEBBBD41C5D26BF1ull), P5 = dfromb(0x3E66376972BEA4D0ull);
  uint32_t hx = hiword(x);
  const int sign = (int)(hx >> 31);
  hx &= 0x7fffffffu;
  if (hx >= 0x4086232bu) {                                   // |x| >= 708.39...
    if (x != x) return x;
    if (x > 709.782712893383973096) return x * dfromb(0x7fe0000000000000ull);   // overflow (inf stays inf)
    if (x < -745.13321910194110842) return 0.0;              // underflow (x < -708.39... otherwise goes on to the subnormal result)
  }
  double hi, lo; int k;
  if (hx > 0x3fd62e42u) {                                    // |x| > ln2 / 2
    if (hx >= 0x3ff0a2b2u) k = (int)(INVLN2 * x + (sign ? -0.5 : 0.5));   // |x| >= 1.5 ln2
    else k = 1 - sign - sign;
    hi = x - (double)k * LN2HI;                              // exact
    lo = (double)k * LN2LO;
    x = hi - lo;
  } else if (hx > 0x3e300000u) {                             // |x| > 2^-28
    k = 0; hi = x; lo = 0.0;
  } else {
    return 1.0 + x;
  }
  const double xx = x * x;
  const double c = x - xx * (P1 + xx * (P2 + xx * (P3 + xx * (P4 + xx * P5))));
  const double y = 1.0 + (x * c / (2.0 - c) - lo + hi);
  return k == 0 ? y : scalbn(y, k);
}

}  // namespace m64

// reference src/svf.rs:26-221 SvfCoefs<f64>: the f32 forms of libm.cuh with F = f64 (PI = f64::PI, libm tan, IEEE sqrt)
struct SvfCoefs64 { double a1, a2, a3, m0, m1, m2; };
template <int MODE> FDSP_HD SvfCoefs64 svf_coefs64(double sr, double cutoff, double q, double gain) {
  const double PI = 3.14159265358979323846;
  SvfCoefs64 c; double g, k;
  if (MODE <= 5) { g = m64::tan(PI * cutoff / sr); k = 1.0 / q; c.m0 = c.m1 = c.m2 = 0.0; }
  else if (MODE == 6) { double a = sqrt(gain); g = m64::tan(PI * cutoff / sr); k = 1.0 / (q * a); c.m0 = 1.0; c.m1 = k * (a * a - 1.0); c.m2 = 0.0; }
  else if (MODE == 7) { double a = sqrt(gain); g = m64::tan(PI * cutoff / sr) / sqrt(a); k = 1.0 / q; c.m0 = 1.0; c.m1 = k * (a - 1.0); c.m2 = a * a - 1.0; }
  else { double a = sqrt(gain); g = m64::tan(PI * cutoff / sr) * sqrt(a); k = 1.0 / q; c.m0 = a * a; c.m1 = k * (1.0 - a) * a; c.m2 = 1.0 - a * a; }
  c.a1 = 1.0 / (1.0 + g * (g + k)); c.a2 = g * c.a1; c.a3 = g * c.a2;
  if (MODE == 0) { c.m0 = 0.0; c.m1 = 0.0; c.m2 = 1.0; }
  if (MODE == 1) { c.m0 = 1.0; c.m1 = -k; c.m2 = -1.0; }
  if (MODE == 2) { c.m0 = 0.0; c.m1 = 1.0; c.m2 = 0.0; }
  if (MODE == 3) { c.m0 = 1.0; c.m1 = -k; c.m2 = 0.0; }
  if (MODE == 4) { c.m0 = 1.0; c.m1 = -k; c.m2 = -2.0; }
  if (MODE == 5) { c.m0 = 1.0; c.m1 = -2.0 * k; c.m2 = 0.0; }
  return c;
}

// reference src/biquad.rs:27-50 BiquadCoefs<f64>::butter_lowpass / resonator (F::PI, F::TAU, F::SQRT_2 of f64; libm tan / exp / cos)
struct BqCoefs64 { double a1, a2, b0, b1, b2; };
FDSP_HD BqCoefs64 bq_butter_lowpass64(double sr, double cutoff) {
  const double PI = 3.14159265358979323846, SQRT_2 = 1.41421356237309504880;
  const double f = m64::tan(cutoff * PI / sr);
  const double a0r = 1.0 / (1.0 + SQRT_2 * f + f * f);
  BqCoefs64 c; c.a1 = (2.0 * f * f - 2.0) * a0r; c.a2 = (1.0 - SQRT_2 * f + f * f) * a0r;
  c.b0 = f * f * a0r; c.b1 = 2.0 * c.b0; c.b2 = c.b0; return c;
}
FDSP_HD BqCoefs64 bq_resonator64(double sr, double center, double q) {
  const double PI = 3.14159265358979323846, TAU = 6.28318530717958647693;
  const double r = m64::exp(-PI * center / (q * sr));
  BqCoefs64 c; c.a1 = -2.0 * r * m64::cos(TAU * center / sr); c.a2 = r * r;
  c.b0 = sqrt(1.0 - r * r) * 0.5; c.b1 = 0.0; c.b2 = -c.b0; return c;
}
// reference src/filter.rs with F = f64: Lowpole / Highpole exp(-TAU cutoff / sr) (:43-46, :376-379), Allpole (1 - d) / (1 + d) (:294-296),
// DCBlock 1 - TAU / sr * cutoff (:123-126); kind as in OnePole64
FDSP_HD double onepole_coeff64(int kind, double sr, double p) {
  const double TAU = 6.28318530717958647693;
  if (kind == 0 || kind == 1) return m64::exp(-TAU * p / sr);
  if (kind == 2) return (1.0 - p) / (1.0 + p);
  return 1.0 - TAU / sr * p;
}

}  // namespace fdsp

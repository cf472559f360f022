// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h). The f64 sin/cos/tan/exp that the reference's f64 nodes call (reference
// src/lib.rs:520-568 -> the Rust `libm` crate, a port of musl / FreeBSD msun), restated independently of the product's
// csrc/dsp/libm64.cuh: word access through unions, k_tan in FreeBSD's `iy = +-1` form, the near-multiples of pi/2 from a table,
// and exp's final scaling by std::ldexp (correctly rounded, like the crate's scalbn). Arguments with |x| >= 2^20 pi/2 are reduced by
// k_rem_pio2.c's Payne-Hanek path at prec 1, restated below with its own digits of 2/pi: no trig path calls the C library's functions.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace fo {
namespace m64 {

union DW { double d; uint64_t u; struct { uint32_t lo, hi; } w; };
inline uint32_t high_word(double x) { DW v; v.d = x; return v.w.hi; }
inline double with_low_word(double x, uint32_t lo) { DW v; v.d = x; v.w.lo = lo; return v.d; }
inline double hexd(uint32_t hi, uint32_t lo) { DW v; v.w.hi = hi; v.w.lo = lo; return v.d; }

inline double kernel_sin(double x, double y, int iy) {
  static const double S[6] = {hexd(0xBFC55555, 0x55555549), hexd(0x3F811111, 0x1110F8A6), hexd(0xBF2A01A0, 0x19C161D5),
                              hexd(0x3EC71DE3, 0x57B1FE7D), hexd(0xBE5AE5E6, 0x8A2B9CEB), hexd(0x3DE5D93A, 0x5ACFD57C)};
  double z = x * x, w = z * z;
  double r = S[1] + z * (S[2] + z * S[3]) + z * w * (S[4] + z * S[5]);
  double v = z * x;
  if (iy == 0) return x + v * (S[0] + z * r);
  return x - ((z * (0.5 * y - v * r) - y) - v * S[0]);
}
inline double kernel_cos(double x, double y) {
  static const double C[6] = {hexd(0x3FA55555, 0x5555554C), hexd(0xBF56C16C, 0x16C15177), hexd(0x3EFA01A0, 0x19CB1590),
                              hexd(0xBE927E4F, 0x809C52AD), hexd(0x3E21EE9E, 0xBDB4B1C4), hexd(0xBDA8FAE9, 0xBE8838D4)};
  double z = x * x, w = z * z;
  double r = z * (C[0] + z * (C[1] + z * C[2])) + w * w * (C[3] + z * (C[4] + z * C[5]));
  double hz = 0.5 * z;
  w = 1.0 - hz;
  return w + (((1.0 - w) - hz) + (z * r - x * y));
}
// FreeBSD k_tan.c: iy = 1 gives tan(x + y), iy = -1 gives -1 / tan(x + y)
inline double kernel_tan(double x, double y, int iy) {
  static const double T[13] = {
      hexd(0x3FD55555, 0x55555563), hexd(0x3FC11111, 0x1110FE7A), hexd(0x3FABA1BA, 0x1BB341FE), hexd(0x3F9664F4, 0x8406D637),
      hexd(0x3F8226E3, 0xE96E8493), hexd(0x3F6D6D22, 0xC9560328), hexd(0x3F57DBC8, 0xFEE08315), hexd(0x3F4344D8, 0xF2F26501),
      hexd(0x3F3026F7, 0x1A8D1068), hexd(0x3F147E88, 0xA03792A6), hexd(0x3F12B80F, 0x32F0A7E9), hexd(0xBEF375CB, 0xDB605373),
      hexd(0x3EFB2A70, 0x74BF7AD4)};
  const double pio4 = hexd(0x3FE921FB, 0x54442D18), pio4lo = hexd(0x3C81A626, 0x33145C07);
  const int32_t hx = (int32_t)high_word(x);
  const int32_t ix = hx & 0x7fffffff;
  if (ix >= 0x3FE59428) {
    if (hx < 0) { x = -x; y = -y; }
    double z = pio4 - x, w = pio4lo - y;
    x = z + w; y = 0.0;
  }
  double z = x * x, w = z * z;
  double r = T[1] + w * (T[3] + w * (T[5] + w * (T[7] + w * (T[9] + w * T[11]))));
  double v = z * (T[2] + w * (T[4] + w * (T[6] + w * (T[8] + w * (T[10] + w * T[12])))));
  double s = z * x;
  r = y + z * (s * (r + v) + y);
  r += T[0] * s;
  w = x + r;
  if (ix >= 0x3FE59428) {
    v = (double)iy;
    return (double)(1 - ((hx >> 30) & 2)) * (v - 2.0 * (x - (w * w / (w + v) - r)));
  }
  if (iy == 1) return w;
  double a, t;
  z = with_low_word(w, 0);
  v = r - (z - x);
  t = a = -1.0 / w;
  t = with_low_word(t, 0);
  s = 1.0 + t * z;
  return t + a * (s + t * v);
}

// e_rem_pio2.c for |x| < 2^20 pi/2 (rem_pio2_big takes the rest); returns n with x = n pi/2 + y[0] + y[1]
inline int rem_pio2(double x, double* y) {
  const double invpio2 = hexd(0x3FE45F30, 0x6DC9C883), pio2_1 = hexd(0x3FF921FB, 0x54400000), pio2_1t = hexd(0x3DD0B461, 0x1A626331),
               pio2_2 = hexd(0x3DD0B461, 0x1A600000), pio2_2t = hexd(0x3BA3198A, 0x2E037073), pio2_3 = hexd(0x3BA3198A, 0x2E000000),
               pio2_3t = hexd(0x397B839A, 0x252049C1);
  const int32_t hx = (int32_t)high_word(x), ix = hx & 0x7fffffff;
  // the one-round cases: upper bound of |x|'s high word for n = 1..4, and the high words that take the medium path instead
  static const int32_t bound[4] = {0x4002d97c, 0x400f6a7a, 0x4015fdbc, 0x401c463b};
  const bool medium = ix > 0x401c463b || (ix <= 0x400f6a7a && (ix & 0xfffff) == 0x921fb) || ix == 0x4012d97c || ix == 0x401921fb;
  if (!medium) {
    int n = 1;
    while (ix > bound[n - 1]) n++;
    const double p = n * pio2_1, pt = n * pio2_1t;
    if (hx > 0) { double z = x - p; y[0] = z - pt; y[1] = (z - y[0]) - pt; return n; }
    double z = x + p; y[0] = z + pt; y[1] = (z - y[0]) + pt; return -n;
  }
  double fn = (x * invpio2 + 0x1.8p52) - 0x1.8p52;
  int n = (int)fn;
  double r = x - fn * pio2_1, w = fn * pio2_1t;
  int j = ix >> 20;
  y[0] = r - w;
  int i = j - (int)((high_word(y[0]) >> 20) & 0x7ff);
  if (i > 16) {
    double t = r;
    w = fn * pio2_2; r = t - w; w = fn * pio2_2t - ((t - r) - w);
    y[0] = r - w;
    i = j - (int)((high_word(y[0]) >> 20) & 0x7ff);
    if (i > 49) {
      t = r;
      w = fn * pio2_3; r = t - w; w = fn * pio2_3t - ((t - r) - w);
      y[0] = r - w;
    }
  }
  y[1] = (r - y[0]) - w;
  return n;
}

// k_rem_pio2.c __rem_pio2_large(x, y, e0, nx, prec) for prec 1 (init_jk[1] = 4, two doubles out): x[0..nx-1] are 24-bit pieces of
// |arg| 2^-e0, y[0] + y[1] = |arg| - n pi/2 with n returned mod 8.
// 2/pi to 1584 bits: 66 digits of 24 bits, the 41 + 4 that the largest double's e0 = 1000 reads at once plus room for recomputation.
static const char TWO_OVER_PI_HEX[] =
    "a2f9836e4e441529fc2757d1f534ddc0db6295993c439041fe5163abdebbc561b7246e3a424dd2e006492eea09d1921cfe1deb1cb129a73ee88235f5"
    "2ebb4484e99c7026b45f7e413991d639835339f49c845f8bbdf9283b1ff897ffde05980fef2f118b5a0a6d1f6d367ecf27cb09b74f463f669e5fea2d"
    "7527bac7ebe5f17b3d0739f78a5292ea6bfb5fb11f8d5d0856033046fc7b6babf0cfbc209af4361da9e391615ee61b086599855f14a068408dffd880"
    "4d73273106061556ca73a8c960e27bc08c6b";
const int TWO_OVER_PI_DIGITS = (int)(sizeof(TWO_OVER_PI_HEX) - 1) / 6;
inline int32_t two_over_pi_digit(int k) {   // 24 bits k of the fraction of 2/pi: hex digits 6k .. 6k + 5
  int32_t d = 0;
  for (int h = 6 * k; h < 6 * k + 6; h++) {
    const char c = TWO_OVER_PI_HEX[h];
    d = d * 16 + (c <= '9' ? c - '0' : c - 'a' + 10);
  }
  return d;
}
inline int rem_pio2_large(const double* x, double* y, int e0, int nx) {
  static const double PIo2[5] = {1.57079625129699707031e+00, 7.54978941586159635335e-08, 5.39030252995776476554e-15,
                                 3.28200341580791294123e-22, 1.27065575308067607349e-29};
  const int jk = 4, jp = jk;
  int32_t jz, jx, jv, carry, n, iq[20], i, j, k, m, q0, ih;
  double z, fw, f[20], fq[20], q[20];
  jx = nx - 1;
  jv = (e0 - 3) / 24; if (jv < 0) jv = 0;
  q0 = e0 - 24 * (jv + 1);
  j = jv - jx; m = jx + jk;
  for (i = 0; i <= m; i++, j++) f[i] = j < 0 ? 0.0 : (double)two_over_pi_digit(j);
  for (i = 0; i <= jk; i++) { for (j = 0, fw = 0.0; j <= jx; j++) fw += x[j] * f[jx + i - j]; q[i] = fw; }
  jz = jk;
recompute:
  for (i = 0, j = jz, z = q[jz]; j > 0; i++, j--) {
    fw = (double)(int32_t)(0x1p-24 * z);
    iq[i] = (int32_t)(z - 0x1p24 * fw);
    z = q[j - 1] + fw;
  }
  z = std::ldexp(z, q0);
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
    if (ih == 2) { z = 1.0 - z; if (carry != 0) z -= std::ldexp(1.0, q0); }
  }
  if (z == 0) {
    j = 0;
    for (i = jz - 1; i >= jk; i--) j |= iq[i];
    if (j == 0) {
      for (k = 1; iq[jk - k] == 0; k++) {}
      for (i = jz + 1; i <= jz + k; i++) {
        f[jx + i] = (double)two_over_pi_digit(jv + i);
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
    z = std::ldexp(z, -q0);
    if (z >= 0x1p24) {
      fw = (double)(int32_t)(0x1p-24 * z);
      iq[jz] = (int32_t)(z - 0x1p24 * fw);
      jz += 1; q0 += 24;
      iq[jz] = (int32_t)fw;
    } else iq[jz] = (int32_t)z;
  }
  fw = std::ldexp(1.0, q0);
  for (i = jz; i >= 0; i--) { q[i] = fw * (double)iq[i]; fw *= 0x1p-24; }
  for (i = jz; i >= 0; i--) {
    for (fw = 0.0, k = 0; k <= jp && k <= jz - i; k++) fw += PIo2[k] * q[i + k];
    fq[jz - i] = fw;
  }
  fw = 0.0;
  for (i = jz; i >= 0; i--) fw += fq[i];
  y[0] = ih == 0 ? fw : -fw;
  fw = fq[0] - fw;
  for (i = 1; i <= jz; i++) fw += fq[i];
  y[1] = ih == 0 ? fw : -fw;
  return n & 7;
}
// e_rem_pio2.c's large case for finite x: |x| 2^-e0 in [2^23, 2^24) split into three 24-bit pieces, trailing zero pieces dropped
inline int rem_pio2_big(double x, double* y) {
  const int e0 = std::ilogb(x) - 23;
  double z = std::ldexp(std::fabs(x), -e0), tx[3];
  for (int i = 0; i < 2; i++) { tx[i] = std::trunc(z); z = (z - tx[i]) * 0x1p24; }
  tx[2] = z;
  int nx = 3;
  while (nx > 1 && tx[nx - 1] == 0.0) nx--;
  double ty[2];
  const int n = rem_pio2_large(tx, ty, e0, nx);
  if (std::signbit(x)) { y[0] = -ty[0]; y[1] = -ty[1]; return -n; }
  y[0] = ty[0]; y[1] = ty[1];
  return n;
}
// any finite x: the medium reduction below 2^20 pi/2, the large one above
inline int rem_pio2_any(double x, double* y) {
  return (int32_t)(high_word(x) & 0x7fffffff) >= 0x413921fb ? rem_pio2_big(x, y) : rem_pio2(x, y);
}

inline double sin(double x) {
  const int32_t ix = (int32_t)(high_word(x) & 0x7fffffff);
  if (ix <= 0x3fe921fb) return ix < 0x3e500000 ? x : kernel_sin(x, 0.0, 0);
  if (ix >= 0x7ff00000) return x - x;
  double y[2]; const int n = rem_pio2_any(x, y);
  switch (n & 3) {
    case 0: return kernel_sin(y[0], y[1], 1);
    case 1: return kernel_cos(y[0], y[1]);
    case 2: return -kernel_sin(y[0], y[1], 1);
    default: return -kernel_cos(y[0], y[1]);
  }
}
inline double cos(double x) {
  const int32_t ix = (int32_t)(high_word(x) & 0x7fffffff);
  if (ix <= 0x3fe921fb) return ix < 0x3e46a09e ? 1.0 : kernel_cos(x, 0.0);
  if (ix >= 0x7ff00000) return x - x;
  double y[2]; const int n = rem_pio2_any(x, y);
  switch (n & 3) {
    case 0: return kernel_cos(y[0], y[1]);
    case 1: return -kernel_sin(y[0], y[1], 1);
    case 2: return -kernel_cos(y[0], y[1]);
    default: return kernel_sin(y[0], y[1], 1);
  }
}
inline double tan(double x) {
  const int32_t ix = (int32_t)(high_word(x) & 0x7fffffff);
  if (ix <= 0x3fe921fb) return ix < 0x3e400000 ? x : kernel_tan(x, 0.0, 1);
  if (ix >= 0x7ff00000) return x - x;
  double y[2]; const int n = rem_pio2_any(x, y);
  return kernel_tan(y[0], y[1], 1 - ((n & 1) << 1));
}
// musl e_exp.c (the crate's exp.rs): reduce x = k ln2 + r, |r| <= ln2 / 2, rational approximation of exp(r), then scale by 2^k
inline double exp(double x) {
  const double ln2hi = hexd(0x3fe62e42, 0xfee00000), ln2lo = hexd(0x3dea39ef, 0x35793c76), invln2 = hexd(0x3ff71547, 0x652b82fe);
  const double P[5] = {hexd(0x3FC55555, 0x5555553E), hexd(0xBF66C16C, 0x16BEBD93), hexd(0x3F11566A, 0xAF25DE2C), hexd(0xBEBBBD41, 0xC5D26BF1),
                       hexd(0x3E663769, 0x72BEA4D0)};
  const uint32_t hw = high_word(x), hx = hw & 0x7fffffff;
  const int sign = (int)(hw >> 31);
  if (hx >= 0x4086232b) {
    if (std::isnan(x)) return x;
    if (x > 709.782712893383973096) return x * 0x1p1023;
    if (x < -745.13321910194110842) return 0.0;
  }
  double hi = 0.0, lo = 0.0; int k = 0;
  if (hx > 0x3fd62e42) {
    k = hx >= 0x3ff0a2b2 ? (int)(invln2 * x + (sign ? -0.5 : 0.5)) : (sign ? -1 : 1);
    hi = x - k * ln2hi;
    lo = k * ln2lo;
    x = hi - lo;
  } else if (hx > 0x3e300000) {
    hi = x;
  } else {
    return 1.0 + x;
  }
  const double xx = x * x;
  const double c = x - xx * (P[0] + xx * (P[1] + xx * (P[2] + xx * (P[3] + xx * P[4]))));
  const double y = 1.0 + (x * c / (2.0 - c) - lo + hi);
  return k == 0 ? y : std::ldexp(y, k);
}

}  // namespace m64
}  // namespace fo

// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h). The f64 sin/cos/tan/exp that the reference's f64 nodes call (reference
// src/lib.rs:520-568 -> the Rust `libm` crate, a port of musl / FreeBSD msun), restated independently of the product's
// csrc/dsp/libm64.cuh: word access through unions, k_tan in FreeBSD's `iy = +-1` form, the near-multiples of pi/2 from a table,
// and exp's final scaling by std::ldexp (correctly rounded, like the crate's scalbn). Arguments with |x| >= 2^20 pi/2 use the C
// library's functions (msun's k_rem_pio2.c is not restated; the product does the same).
#pragma once
#include <cmath>
#include <cstdint>

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

// e_rem_pio2.c for |x| < 2^20 pi/2; returns n with x = n pi/2 + y[0] + y[1]
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

inline double sin(double x) {
  const int32_t ix = (int32_t)(high_word(x) & 0x7fffffff);
  if (ix <= 0x3fe921fb) return ix < 0x3e500000 ? x : kernel_sin(x, 0.0, 0);
  if (ix >= 0x7ff00000) return x - x;
  if (ix >= 0x413921fb) return std::sin(x);
  double y[2]; const int n = rem_pio2(x, y);
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
  if (ix >= 0x413921fb) return std::cos(x);
  double y[2]; const int n = rem_pio2(x, y);
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
  if (ix >= 0x413921fb) return std::tan(x);
  double y[2]; const int n = rem_pio2(x, y);
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

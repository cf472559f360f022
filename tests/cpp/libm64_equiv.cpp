// TEST INFRASTRUCTURE: the PRODUCT's f64 sin/cos/tan/exp (fundsp_b200/csrc/dsp/libm64.cuh), compiled for the host through the
// FDSP_HOST_EMUL shims, against the ORACLE's independent restatement (oracle/fo_libm64.h), bit for bit, and (built with -DFO_QUAD and
// libquadmath) both against the __float128 functions, in ulps of the f64 result.
//   g++ -std=c++17 -O2 -ffp-contract=off -pthread -DFO_QUAD tests/cpp/libm64_equiv.cpp -o libm64_equiv -l:libquadmath.so.0
//   ./libm64_equiv HI_STRIDE DENSE
// HI_STRIDE: every HI_STRIDE-th high word (1 = all 2^32) with the low words 0, 1, 0x80000000, 0xffffffff. DENSE: points evenly spread
// over the domains the filters use (tan on [0, pi/2), cos on [0, 2 pi], exp on [-746, 710]); 0 skips them. The special values are
// always checked. Output: per function "<name>: N mismatches" (plus the first), "<name>: max ulp E at x", and "specials: ok|FAIL".
#define FDSP_HOST_EMUL 1
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <thread>
#include <vector>

#include "../../fundsp_b200/csrc/dsp/libm64.cuh"
#include "../../oracle/fo_libm64.h"
#ifdef FO_QUAD
#include <quadmath.h>
#endif

static inline uint64_t b64(double x) { uint64_t u; memcpy(&u, &x, 8); return u; }
static inline double d64(uint64_t u) { double x; memcpy(&x, &u, 8); return x; }
static inline bool same(double a, double b) { return (a != a && b != b) || b64(a) == b64(b); }

static double prod(int f, double x) { switch (f) { case 0: return fdsp::m64::sin(x); case 1: return fdsp::m64::cos(x); case 2: return fdsp::m64::tan(x); default: return fdsp::m64::exp(x); } }
static double orac(int f, double x) { switch (f) { case 0: return fo::m64::sin(x); case 1: return fo::m64::cos(x); case 2: return fo::m64::tan(x); default: return fo::m64::exp(x); } }
// where a function's accuracy is the restatement's own (the trig functions hand |x| >= 2^20 pi/2 to the C library)
static bool own(int f, double x) { return std::isfinite(x) && (f == 3 || std::fabs(x) < 1647099.3291652855); }
#ifdef FO_QUAD
static double ulps(int f, double y, double x) {
  const __float128 q = x;
  const __float128 e = f == 0 ? sinq(q) : f == 1 ? cosq(q) : f == 2 ? tanq(q) : expq(q);
  if (y != y) return 1e30;
  const double r = std::fabs((double)e);
  if (r == INFINITY) return std::isinf(y) ? 0.0 : 1e30;
  const double sp = r < 2.2250738585072014e-308 ? std::ldexp(1.0, -1074) : std::nextafter(r, INFINITY) - r;
  return (double)fabsq((__float128)y - e) / sp;
}
#endif

int main(int argc, char** argv) {
  const uint64_t hstride = argc > 1 ? strtoull(argv[1], nullptr, 10) : 97;
  const uint64_t dense = argc > 2 ? strtoull(argv[2], nullptr, 10) : 0;
  const unsigned nt = std::max(1u, std::thread::hardware_concurrency());
  const uint32_t lows[4] = {0u, 1u, 0x80000000u, 0xffffffffu};
  const double lo[4] = {0.0, 0.0, 0.0, -746.0}, hi[4] = {0.0, 2.0 * 3.14159265358979323846, 3.14159265358979323846 / 2.0, 710.0};
  std::vector<uint64_t> bad(nt * 4, 0), first(nt * 4, 0);
  std::vector<double> worst(nt * 4, 0.0), worst_x(nt * 4, 0.0);
  auto check = [&](unsigned t, int f, double x, bool acc) {
    const double p = prod(f, x), o = orac(f, x);
    if (!same(p, o)) { if (!bad[t * 4 + f]) first[t * 4 + f] = b64(x); bad[t * 4 + f]++; }
#ifdef FO_QUAD
    if (acc && own(f, x)) { const double e = ulps(f, p, x); if (e > worst[t * 4 + f]) { worst[t * 4 + f] = e; worst_x[t * 4 + f] = x; } }
#else
    (void)acc;
#endif
  };
  std::vector<std::thread> th;
  for (unsigned t = 0; t < nt; t++) th.emplace_back([&, t] {
    uint64_t k = 0;
    for (uint64_t h = t * hstride; h < (1ull << 32); h += (uint64_t)nt * hstride)
      for (uint32_t l : lows) {
        const double x = d64((h << 32) | l);
        k++;
        for (int f = 0; f < 4; f++) check(t, f, x, (k & 1023) == 0);
      }
    for (int f = 1; f < 4; f++)   // sin is not a filter function: the high-word sweep covers it
      for (uint64_t i = t; i < dense; i += nt) {
        double x = lo[f] + (hi[f] - lo[f]) * ((double)i / (double)dense);
        if (f == 2 && x >= hi[f]) continue;
        check(t, f, x, (i & 63) == 0);
      }
  });
  for (auto& x : th) x.join();
  const char* names[4] = {"sin", "cos", "tan", "exp"};
  int rc = 0;
  for (int f = 0; f < 4; f++) {
    uint64_t b = 0, fi = 0; double w = 0.0, wx = 0.0;
    for (unsigned t = 0; t < nt; t++) {
      b += bad[t * 4 + f]; if (bad[t * 4 + f] && !fi) fi = first[t * 4 + f];
      if (worst[t * 4 + f] > w) { w = worst[t * 4 + f]; wx = worst_x[t * 4 + f]; }
    }
    printf("%s: %llu mismatches%s\n", names[f], (unsigned long long)b, b ? "" : " (bit-identical)");
    if (b) { printf("  first at bits 0x%016llx\n", (unsigned long long)fi); rc = 1; }
#ifdef FO_QUAD
    printf("%s: max ulp %.4f at x = %.17g\n", names[f], w, wx);
#endif
  }
  // special values: signed zeros, subnormals, infinities, NaN, exp's overflow and underflow thresholds
  bool ok = true;
  const double dmin = d64(1), nan = d64(0x7ff8000000000000ull);
  for (int f = 0; f < 4; f++)
    for (double x : {0.0, -0.0, dmin, -dmin, d64(0x000fffffffffffffull), (double)INFINITY, -(double)INFINITY, nan, 709.782712893383973096, 709.7827128933841,
                     -745.13321910194110842, -745.1332191019412, -708.39641853226410622, -740.0})
      ok = ok && same(prod(f, x), orac(f, x));
  using fdsp::m64::sin; using fdsp::m64::cos; using fdsp::m64::tan; using fdsp::m64::exp;
  ok = ok && b64(sin(-0.0)) == b64(-0.0) && b64(tan(-0.0)) == b64(-0.0) && cos(-0.0) == 1.0 && sin(dmin) == dmin && tan(-dmin) == -dmin;
  ok = ok && std::isnan(sin(INFINITY)) && std::isnan(cos(-INFINITY)) && std::isnan(tan(INFINITY)) && std::isnan(sin(nan)) && std::isnan(exp(nan));
  ok = ok && exp(INFINITY) == INFINITY && exp(-INFINITY) == 0.0 && exp(0.0) == 1.0 && exp(-0.0) == 1.0;
  ok = ok && std::isfinite(exp(709.782712893383973096)) && exp(709.7827128933841) == INFINITY;   // the largest finite result, then overflow
  ok = ok && exp(-745.13321910194110842) > 0.0 && exp(-745.1332191019412) == 0.0;               // the smallest subnormal, then zero
  ok = ok && exp(-740.0) > 0.0 && exp(-740.0) < 2.2250738585072014e-308;                         // a subnormal result
  printf("specials: %s\n", ok ? "ok" : "FAIL");
  return rc || !ok;
}

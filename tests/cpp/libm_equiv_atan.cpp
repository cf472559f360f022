// TEST INFRASTRUCTURE: the PRODUCT's atanf_ (fundsp_b200/csrc/dsp/libm.cuh) and wide_atanf (math.cuh), compiled for the host through the
// FDSP_HOST_EMUL shims, against the ORACLE's independent restatements (oracle/fo_shapes.h), bit for bit over float bit patterns, and
// both against the float64 arctan, in ulps of the f32 result.
//   g++ -std=c++17 -O2 -ffp-contract=off -pthread tests/cpp/libm_equiv_atan.cpp -o libm_equiv_atan ; ./libm_equiv_atan STRIDE   (1 = all 2^32)
// NaNs compare as a class. Output: one "<name>: N mismatches" line per function, then "<name>: max ulp E at bits 0x...".
#define FDSP_HOST_EMUL 1
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <thread>
#include <vector>

#include "../../fundsp_b200/csrc/dsp/libm.cuh"
#include "../../oracle/fo_shapes.h"

static inline float fromb_(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t bits_(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline bool same(float a, float b) { return (a != a && b != b) || bits_(a) == bits_(b); }
// |y - exact| in units of the f32 spacing at |exact| (the spacing of the binade the correctly rounded result lies in)
static inline double ulps(float y, double exact) {
  if (y != y || exact != exact) return (y != y && exact != exact) ? 0.0 : 1e30;
  const float r = std::fabs((float)exact);
  const double sp = r < 1.1754943508222875e-38f ? std::ldexp(1.0, -149) : (double)std::nextafter(r, INFINITY) - (double)r;
  return std::fabs((double)y - exact) / sp;
}

int main(int argc, char** argv) {
  const uint64_t stride = argc > 1 ? strtoull(argv[1], nullptr, 10) : 257;
  const unsigned nt = std::max(1u, std::thread::hardware_concurrency());
  std::vector<uint64_t> bad(nt * 2, 0), first(nt * 2, 0), worst_at(nt * 2, 0);
  std::vector<double> worst(nt * 2, 0.0);
  std::vector<std::thread> th;
  for (unsigned t = 0; t < nt; t++) th.emplace_back([&, t] {
    for (uint64_t u = t * stride; u < (1ull << 32); u += (uint64_t)nt * stride) {
      const float x = fromb_((uint32_t)u);
      const float p[2] = {fdsp::m::atanf_(x), fdsp::wide_atanf(x)};
      const float o[2] = {fo::m::atanf_(x), fo::wide_atanf(x)};
      const double exact = std::atan((double)x);
      for (int k = 0; k < 2; k++) {
        if (!same(p[k], o[k])) { if (!bad[t * 2 + k]) first[t * 2 + k] = u; bad[t * 2 + k]++; }
        const double e = ulps(p[k], exact);
        if (e > worst[t * 2 + k]) { worst[t * 2 + k] = e; worst_at[t * 2 + k] = u; }
      }
    }
  });
  for (auto& x : th) x.join();
  const char* names[2] = {"atanf", "wide_atanf"};
  int rc = 0;
  for (int k = 0; k < 2; k++) {
    uint64_t b = 0, f = 0, wa = 0; double w = 0.0;
    for (unsigned t = 0; t < nt; t++) {
      b += bad[t * 2 + k]; if (bad[t * 2 + k] && !f) f = first[t * 2 + k];
      if (worst[t * 2 + k] > w) { w = worst[t * 2 + k]; wa = worst_at[t * 2 + k]; }
    }
    printf("%s: %llu mismatches%s\n", names[k], (unsigned long long)b, b ? "" : " (bit-identical)");
    if (b) { printf("  first at bits 0x%08llx\n", (unsigned long long)f); rc = 1; }
    printf("%s: max ulp %.4f at bits 0x%08llx\n", names[k], w, (unsigned long long)wa);
  }
  return rc;
}

// TEST INFRASTRUCTURE: the PRODUCT's f64 trig functions and argument reductions (fundsp_b200/csrc/dsp/libm64.cuh) at given arguments,
// compiled for the host through the FDSP_HOST_EMUL shims, for tests/test_libm64_sweep_cpu.py to hold against mpmath and the oracle.
//   g++ -std=c++17 -O2 -ffp-contract=off tests/cpp/libm64_points.cpp -o libm64_points
//   libm64_points < ARGS      one argument per line as 16 hex digits of its bit pattern; per argument one line of hex bit patterns:
//                             sin cos tan, n y0 y1 of rem_pio2_large, and n y0 y1 of rem_pio2_medium when |x| < 2^20 pi/2
#define FDSP_HOST_EMUL 1
#include <cinttypes>
#include <cstdio>

#include "../../fundsp_b200/csrc/dsp/libm64.cuh"

int main() {
  using fdsp::m64::dbits; using fdsp::m64::dfromb; using fdsp::m64::hiword; using fdsp::m64::Rem;
  uint64_t u;
  while (scanf("%" SCNx64, &u) == 1) {
    const double x = dfromb(u);
    printf("%016" PRIx64 " %016" PRIx64 " %016" PRIx64, dbits(fdsp::m64::sin(x)), dbits(fdsp::m64::cos(x)), dbits(fdsp::m64::tan(x)));
    const Rem l = fdsp::m64::rem_pio2_large(x);
    printf(" %d %016" PRIx64 " %016" PRIx64, l.n, dbits(l.y0), dbits(l.y1));
    const uint32_t ix = hiword(x) & 0x7fffffffu;
    if (ix < 0x413921fbu) {
      const Rem m = fdsp::m64::rem_pio2_medium(x, ix);
      printf(" %d %016" PRIx64 " %016" PRIx64, m.n, dbits(m.y0), dbits(m.y1));
    }
    printf("\n");
  }
  return 0;
}

// TEST INFRASTRUCTURE: the PRODUCT's powf_ (fundsp_b200/csrc/dsp/libm.cuh, compiled for the host through the FDSP_HOST_EMUL shims)
// against the ORACLE's independent restatement (oracle/fo_libm.h), bit for bit, over the three powf sets of the scalar-math sweep
// (tests/golden/libm_sweep_args.h): every 512th x against 32 y values, every 512th y against 32 x values, and 2^28 hashed pairs.
//   g++ -std=c++17 -O2 -ffp-contract=off -pthread tests/cpp/libm_equiv_pow.cpp -o libm_equiv_pow ; ./libm_equiv_pow [STRIDE]
// (STRIDE 1, the default, walks every pair of the three sets.) NaNs compare as a class.
#define FDSP_HOST_EMUL 1
#include <cstdio>
#include <cstdlib>
#include <thread>
#include <vector>

#include "../../fundsp_b200/csrc/dsp/libm.cuh"
#include "../../oracle/fo_libm.h"
#include "../golden/libm_sweep_args.h"

static inline float fromb_(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t bits_(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline bool same(float a, float b) { return (a != a && b != b) || bits_(a) == bits_(b); }

int main(int argc, char** argv) {
  const uint64_t stride = argc > 1 ? strtoull(argv[1], nullptr, 10) : 1;
  const unsigned nt = std::max(1u, std::thread::hardware_concurrency());
  const int sets[3] = {sweep::POW_X, sweep::POW_Y, sweep::POW_RAND};
  const char* names[] = SWEEP_NAMES;
  int rc = 0;
  for (int s : sets) {
    const uint64_t n = (uint64_t)sweep::chunks(s) << sweep::CHUNK_LOG2;
    std::vector<uint64_t> bad(nt, 0), first(nt, ~0ull), done(nt, 0);
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nt; t++) th.emplace_back([&, t] {
      for (uint64_t i = t * stride; i < n; i += (uint64_t)nt * stride) {
        uint32_t xb, yb;
        sweep::arg_bits(s, i, xb, yb);
        const float x = fromb_(xb), y = fromb_(yb);
        if (!same(fdsp::m::powf_(x, y), fo::m::powf_(x, y))) { if (!bad[t]) first[t] = i; bad[t]++; }
        done[t]++;
      }
    });
    for (auto& x : th) x.join();
    uint64_t b = 0, f = ~0ull, d = 0;
    for (unsigned t = 0; t < nt; t++) { b += bad[t]; d += done[t]; if (first[t] < f) f = first[t]; }
    printf("%s: %llu pairs, %llu mismatches%s\n", names[s], (unsigned long long)d, (unsigned long long)b, b ? "" : " (bit-identical)");
    if (b) {
      uint32_t xb, yb;
      sweep::arg_bits(s, f, xb, yb);
      printf("  first at index %llu: powf(0x%08x, 0x%08x) product 0x%08x oracle 0x%08x\n", (unsigned long long)f, xb, yb,
             bits_(fdsp::m::powf_(fromb_(xb), fromb_(yb))), bits_(fo::m::powf_(fromb_(xb), fromb_(yb))));
      rc = 1;
    }
  }
  return rc;
}

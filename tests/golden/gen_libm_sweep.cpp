// TEST INFRASTRUCTURE: the expected per-chunk hashes of the scalar-math sweep (tests/golden/libm_sweep_args.h), computed from the
// ORACLE's restatements (oracle/fo_libm.h, fo_math.h, fo_shapes.h) on the host. tests/golden/gen_libm_sweep.py builds and runs it and
// writes tests/golden/libm_sweep.json; tests/test_gpu_libm_sweep.py holds the product's device builds to those hashes, and
// tests/test_libm_sweep_cpu.py regenerates every 16th chunk to catch a change of the math without a new fixture.
//   g++ -std=c++17 -O2 -ffp-contract=off -pthread -Ioracle tests/golden/gen_libm_sweep.cpp -o gen_libm_sweep
//   ./gen_libm_sweep [--every N] [fn ...]     (JSON on stdout; --every N: only chunks c with c % N == 0)
// A full regeneration (every chunk of every function, 9 * 2^32 + 3 * 2^28 evaluations) takes 1 min 48 s on 8 x86-64 cores
// (-O2, one thread per core); the every-16th-chunk check of the CPU suite about a sixteenth of that.
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <thread>
#include <vector>

#include "fo_shapes.h"
#include "libm_sweep_args.h"

static inline float f_of(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t b_of(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

static float eval(int fn, float x, float y) {
  switch (fn) {
    case sweep::SINF: return fo::m::sinf_(x);
    case sweep::COSF: return fo::m::cosf_(x);
    case sweep::TANF: return fo::m::tanf_(x);
    case sweep::TANHF: return fo::m::tanhf_(x);
    case sweep::EXPM1F: return fo::m::expm1f_(x);
    case sweep::EXPF: return fo::m::expf_(x);
    case sweep::ATANF: return fo::m::atanf_(x);
    case sweep::WIDE_SINF: return fo::wide_sinf(x);
    case sweep::WIDE_ATANF: return fo::wide_atanf(x);
    default: return fo::m::powf_(x, y);
  }
}

int main(int argc, char** argv) {
  int every = 1;
  std::vector<int> fns;
  const char* names[] = SWEEP_NAMES;
  for (int a = 1; a < argc; a++) {
    const std::string s = argv[a];
    if (s == "--every" && a + 1 < argc) { every = atoi(argv[++a]); continue; }
    int f = -1;
    for (int k = 0; k < sweep::NFN; k++) if (s == names[k]) f = k;
    if (f < 0) { fprintf(stderr, "unknown function %s\n", s.c_str()); return 2; }
    fns.push_back(f);
  }
  if (fns.empty()) for (int k = 0; k < sweep::NFN; k++) fns.push_back(k);
  struct Task { int fn, chunk; uint64_t hash; };
  std::vector<Task> tasks;
  for (int f : fns) for (int c = 0; c < sweep::chunks(f); c += every) tasks.push_back({f, c, 0});
  std::atomic<size_t> next{0};
  std::vector<std::thread> th;
  const unsigned nt = std::max(1u, std::thread::hardware_concurrency());
  for (unsigned t = 0; t < nt; t++) th.emplace_back([&] {
    for (size_t k; (k = next++) < tasks.size();) {
      Task& T = tasks[k];
      uint64_t h = 0;
      const uint64_t i0 = (uint64_t)T.chunk << sweep::CHUNK_LOG2;
      for (uint64_t i = i0; i < i0 + (1ull << sweep::CHUNK_LOG2); i++) {
        uint32_t xb, yb;
        sweep::arg_bits(T.fn, i, xb, yb);
        h += sweep::term(i, b_of(eval(T.fn, f_of(xb), f_of(yb))));
      }
      T.hash = h;
    }
  });
  for (auto& x : th) x.join();
  printf("{\"chunk_log2\": %d, \"every\": %d, \"functions\": {", sweep::CHUNK_LOG2, every);
  size_t k = 0;
  for (size_t a = 0; a < fns.size(); a++) {
    printf("%s\n  \"%s\": [", a ? "," : "", names[fns[a]]);
    for (int c = 0; c < sweep::chunks(fns[a]); c += every, k++) printf("%s\"%016llx\"", c ? ", " : "", (unsigned long long)tasks[k].hash);
    printf("]");
  }
  printf("\n}}\n");
  return 0;
}

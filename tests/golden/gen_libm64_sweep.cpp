// TEST INFRASTRUCTURE: the expected per-chunk hashes of the f64 math sweep (tests/golden/libm64_sweep_args.h), computed from the ORACLE's
// restatement (oracle/fo_libm64.h) on the host. tests/golden/gen_libm64_sweep.py builds and runs it and writes
// tests/golden/libm64_sweep.json; tests/test_gpu_libm64_sweep.py holds the product's device builds to those hashes, and
// tests/test_libm64_sweep_cpu.py regenerates every 64th chunk to catch a change of the math without a new fixture.
//   g++ -std=c++17 -O2 -ffp-contract=off -pthread -Ioracle -Itests/golden tests/golden/gen_libm64_sweep.cpp -o gen_libm64_sweep
//   ./gen_libm64_sweep [--every N] [--chunk K ...] [fn ...]   (JSON on stdout; --every N: only chunks c with c % N == 0; --chunk K:
//                                                             chunk K as well, in increasing order of chunk)
// A full regeneration (514 chunks of each of the four functions, about 4 x 2^33 evaluations, half of the trig ones on the large
// reduction) takes under 12 minutes on 8 x86-64 cores (-O2, one thread per core); the CPU suite's check of every 64th chunk and the
// special chunk about 1/57 of that.
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <thread>
#include <vector>

#include "fo_libm64.h"
#include "libm64_sweep_args.h"

static inline uint64_t b_of(double x) { uint64_t u; memcpy(&u, &x, 8); return u; }

static double eval(int fn, double x) {
  switch (fn) {
    case sweep64::SIN: return fo::m64::sin(x);
    case sweep64::COS: return fo::m64::cos(x);
    case sweep64::TAN: return fo::m64::tan(x);
    default: return fo::m64::exp(x);
  }
}

int main(int argc, char** argv) {
  int every = 1;
  std::vector<int> fns;
  std::vector<bool> extra(sweep64::CHUNKS, false);
  const char* names[] = SWEEP64_NAMES;
  for (int a = 1; a < argc; a++) {
    const std::string s = argv[a];
    if (s == "--every" && a + 1 < argc) { every = atoi(argv[++a]); continue; }
    if (s == "--chunk" && a + 1 < argc) {
      const int k = atoi(argv[++a]);
      if (k < 0 || k >= sweep64::CHUNKS) { fprintf(stderr, "chunk out of range\n"); return 2; }
      extra[k] = true;
      continue;
    }
    int f = -1;
    for (int k = 0; k < sweep64::NFN; k++) if (s == names[k]) f = k;
    if (f < 0) { fprintf(stderr, "unknown function %s\n", s.c_str()); return 2; }
    fns.push_back(f);
  }
  if (every < 1) { fprintf(stderr, "--every N, N >= 1\n"); return 2; }
  if (fns.empty()) for (int k = 0; k < sweep64::NFN; k++) fns.push_back(k);
  struct Task { int fn, chunk; uint64_t hash; };
  std::vector<Task> tasks;
  auto chosen = [&](int c) { return c % every == 0 || extra[c]; };
  for (int f : fns) for (int c = 0; c < sweep64::CHUNKS; c++) if (chosen(c)) tasks.push_back({f, c, 0});
  std::atomic<size_t> next{0};
  std::vector<std::thread> th;
  const unsigned nt = std::max(1u, std::thread::hardware_concurrency());
  for (unsigned t = 0; t < nt; t++) th.emplace_back([&] {
    for (size_t k; (k = next++) < tasks.size();) {
      Task& T = tasks[k];
      uint64_t h = 0;
      const uint64_t i0 = (uint64_t)T.chunk << sweep64::CHUNK_LOG2;
      for (uint64_t i = i0; i < i0 + sweep64::chunk_len(T.chunk); i++) h += sweep64::term(i, b_of(eval(T.fn, sweep64::as_double(sweep64::arg_bits(T.fn, i)))));
      T.hash = h;
    }
  });
  for (auto& x : th) x.join();
  printf("{\"chunk_log2\": %d, \"every\": %d, \"functions\": {", sweep64::CHUNK_LOG2, every);
  size_t k = 0;
  for (size_t a = 0; a < fns.size(); a++) {
    printf("%s\n  \"%s\": [", a ? "," : "", names[fns[a]]);
    bool first = true;
    for (int c = 0; c < sweep64::CHUNKS; c++)
      if (chosen(c)) { printf("%s\"%016llx\"", first ? "" : ", ", (unsigned long long)tasks[k++].hash); first = false; }
    printf("]");
  }
  printf("\n}}\n");
  return 0;
}

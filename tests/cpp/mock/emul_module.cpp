// TEST INFRASTRUCTURE — one graph class of the mock "GPU" (tests/cpp/mock/registry_mock.cpp): the DEVICE node library compiled for the
// CPU (FDSP_HOST_EMUL) and walked through bank_kernel's per-thread block structure for every voice of a launch, reading and writing
// the same argument block (BankArgs) the real kernel gets. The CTA partial mix is summed in the association of bank_kernel's mix tile
// (128 columns, absent voices as zeros, see cta_partial below), so the mock's mixes carry the same bits the exact model of
// tests/test_gpu_mix.py expects from the GPU (DESIGN.md §4).
// Build: g++ -std=c++17 -O1 -ffp-contract=off -shared -fPIC -DGRAPH='<type expression>' -I fundsp_b200/csrc emul_module.cpp
#define FDSP_HOST_EMUL 1
#include "dsp/nodes.cuh"

#include <vector>

using namespace fdsp;
typedef GRAPH G;

// bank_kernel's CTA partial for one (channel, sample) row of the mix tile: NT = 128 columns, column j = voice b * vpc + j (0.0 where there is
// none); two halves of 64 columns, four accumulators each folding QN = 16 consecutive columns, the odd half starting QN columns further;
// (a0 + a1) + (a2 + a3) per half, low half + high half.
template <class F> static float cta_partial(F col) {
  constexpr int NT = 128, HALF = NT / 2, QN = HALF / 4;
  float s[2];
  for (int h = 0; h < 2; h++) {
    float acc[4];
    for (int q = 0; q < 4; q++) {
      const int c0 = h * HALF + (q * QN + h * QN) % HALF;
      float x = col(c0);
      for (int j = 1; j < QN; j++) x += col(c0 + j);
      acc[q] = x;
    }
    s[h] = (acc[0] + acc[1]) + (acc[2] + acc[3]);
  }
  return s[0] + s[1];
}

extern "C" void fdsp_emul_layout(int* lay) {
  lay[0] = G::IN; lay[1] = G::OUT; lay[2] = G::NP; lay[3] = G::NS; lay[4] = G::NU; lay[5] = WaveKind<G>::value;
}

// per_voice_in != null: voice v reads its OWN input rows per_voice_in + v * voice_stride (+ k * a.in_stride + a.in_offset + t) instead of the
// shared bank input — how the mock runs the reverb stage of a two-stage class on the dry rows of the voices (registry_mock.cpp launch_fdn)
extern "C" int fdsp_emul_launch_ex(const BankArgs* ap, int mode, const float* per_voice_in, uint64_t voice_stride);
extern "C" int fdsp_emul_launch(const BankArgs* ap, int mode) { return fdsp_emul_launch_ex(ap, mode, nullptr, 0); }
extern "C" int fdsp_emul_launch_ex(const BankArgs* ap, int mode, const float* per_voice_in, uint64_t voice_stride) {
  const BankArgs& a = *ap;
  constexpr int IN = G::IN, OUT = G::OUT;
  constexpr bool GROUP = GroupPlan<G>::ok && GroupPlan<G>::code <= 256;   // bank_kernel's FDSP_GROUP_COST
  const uint32_t vpc = a.vpc ? a.vpc : 128u, grid = (a.V + vpc - 1) / vpc;
  if ((mode & 2) && !a.partial) return 1;
  if ((mode & 1) && !a.out) return 2;
  std::vector<float> ys((mode & 2) ? (size_t)a.V * OUT * a.n : 0);   // every voice's outputs, summed in tile order after the walk
  for (uint32_t v = 0; v < a.V; v++) {
    typename G::R r;
    CtxT<false> c;
    c.wt = a.wt; c.tsm = 0u; c.tsm_kind = -1; c.dl = a.dline; c.V = a.V; c.v = v; c.sr = a.sr; c.sd64 = a.sd64; c.sd32 = a.sd32;
    c.rp = a.params; c.rs0 = a.state0; c.ru = a.uniform; c.dl_total = a.dl_floats;
    Loader l{a.params, a.state, a.uniform, a.V, v, 0u, 0u, 0u, 0u};
    G::load(r, l);
    auto emit = [&](int k, uint32_t t, float y) {
      if (mode & 1) a.out[(size_t)(a.row_map[v] + (uint32_t)k) * a.out_stride + a.out_offset + t] = y;
      if (mode & 2) ys[((size_t)v * OUT + k) * a.n + t] = y;
    };
    for (uint32_t t0 = 0; t0 < a.n; t0 += 64) {
      const int nb = (a.n - t0) < 64u ? (int)(a.n - t0) : 64;
      const int nfull = nb & ~7;
      const float* irow = (IN > 0) ? (per_voice_in ? per_voice_in + (size_t)v * voice_stride : a.in) + a.in_offset + t0 : nullptr;
      c.n = nb; c.rem = false;
      for (int g = 0; g < nfull; g += 8) {
        if (GROUP) {
          Fr8<IN> in8; Fr8<OUT> o8;
          for (int k = 0; k < IN; k++) for (int j = 0; j < 8; j++) in8.v[k][j] = irow[(size_t)k * a.in_stride + g + j];
          c.i = g; c.first = true;
          group_step<G>(r, c, in8, o8);
          for (int k = 0; k < OUT; k++) for (int j = 0; j < 8; j++) emit(k, t0 + g + j, o8.v[k][j]);
        } else {
          for (int j = 0; j < 8; j++) {
            Fr<IN> x; Fr<OUT> y;
            for (int k = 0; k < IN; k++) x.v[k] = irow[(size_t)k * a.in_stride + g + j];
            c.i = g + j; c.first = (j == 0);
            G::template step<false>(r, c, x, y);
            for (int k = 0; k < OUT; k++) emit(k, t0 + g + j, y.v[k]);
          }
        }
      }
      G::end_simd(r);
      c.rem = true; c.first = false;
      for (int i = nfull; i < nb; i++) {
        Fr<IN> x; Fr<OUT> y;
        for (int k = 0; k < IN; k++) x.v[k] = irow[(size_t)k * a.in_stride + i];
        c.i = i;
        G::template step<false>(r, c, x, y);
        for (int k = 0; k < OUT; k++) emit(k, t0 + i, y.v[k]);
      }
    }
    Saver s{a.state, a.V, v, 0u};
    G::save(r, s);
  }
  if (mode & 2)
    for (uint32_t b = 0; b < grid; b++)
      for (int k = 0; k < OUT; k++)
        for (uint32_t t = 0; t < a.n; t++)
          a.partial[((size_t)b * OUT + k) * a.n + t] = cta_partial([&](int j) {
            const uint32_t v = b * vpc + (uint32_t)j;
            return ((uint32_t)j < vpc && v < a.V) ? ys[((size_t)v * OUT + k) * a.n + t] : 0.0f;
          });
  if ((mode & 2) && a.ticket) {   // the fused finish of short launches (bank_kernel.cuh): CTA-order left fold into the mix
    for (uint32_t ch = 0; ch < (uint32_t)OUT; ch++)
      for (uint32_t t = 0; t < a.n; t++) {
        float s = a.partial[(size_t)ch * a.n + t];
        for (uint32_t q = 1; q < grid; q++) s += a.partial[((size_t)q * OUT + ch) * a.n + t];
        float* p = a.mix + (size_t)ch * a.mix_stride + a.mix_offset + t;
        *p = a.mix_accumulate ? *p + s : s;
      }
  }
  return 0;
}

// fundsp_b200 host graph implementation — see graph.h. Reference citations per class (paths relative to
// the reference checkout). Coefficient formulas are evaluated in f32 with the host libm exactly where the
// reference evaluates them (constructor / set_sample_rate / Setting), never per sample.
#include "graph.h"
#include "closure.h"
#include "../dsp/libm.cuh"
#include "../dsp/libm64.cuh"

#include <cmath>
#include <limits>
#include <memory>
#include <algorithm>
#include <cassert>

namespace fdsp {
namespace host {

std::vector<uint64_t>*& HNode::ping_trace() { static std::vector<uint64_t>* t = nullptr; return t; }

AttoHash HNode::ping(bool probe, AttoHash hash) {  // src/audionode.rs:156-161
  if (!probe) { set_hash(hash.state); if (ping_trace()) ping_trace()->push_back(hash.state); }
  return hash.hash(id());
}

namespace {

#define HCLONE(T) HNode* clone() const override { return new T(*this); }

struct Kid {  // deep-copying owning pointer
  std::unique_ptr<HNode> p;
  Kid() {}
  explicit Kid(HNode* n) : p(n) {}
  Kid(const Kid& o) : p(o.p ? o.p->clone() : nullptr) {}
  Kid(Kid&& o) noexcept : p(std::move(o.p)) {}
  Kid& operator=(const Kid& o) { if (this != &o) p.reset(o.p ? o.p->clone() : nullptr); return *this; }
  Kid& operator=(Kid&& o) noexcept { p = std::move(o.p); return *this; }
  HNode* operator->() const { return p.get(); }
  HNode& operator*() const { return *p; }
};

std::string I(int v) { return std::to_string(v); }

// ---------------------------------------------------------------- routing leaves (src/audionode.rs:374-722,2800-2837)
struct Routing : HNode {
  enum K { PASS, MULTIPASS, SINK, SPLIT, MULTISPLIT, JOIN, MULTIJOIN, REVERSE, MONITOR } k; int m, n;   // MONITOR: src/dynamics.rs:441 passes its input through (the Shared it feeds is host-side state)
  Routing(K k_, int m_, int n_) : k(k_), m(m_), n(n_) {}
  int inputs() const override {
    switch (k) { case PASS: case MONITOR: return 1; case MULTIPASS: case SINK: case REVERSE: return n; case SPLIT: return 1; case MULTISPLIT: return m;
      case JOIN: return n; default: return m * n; }
  }
  int outputs() const override {
    switch (k) { case PASS: case MONITOR: return 1; case MULTIPASS: case REVERSE: return n; case SINK: return 0; case SPLIT: return n; case MULTISPLIT: return m * n;
      case JOIN: return 1; default: return m; }
  }
  uint64_t id() const override {
    switch (k) { case PASS: return 48; case MONITOR: return 56; case MULTIPASS: return 0; case SINK: return 1; case SPLIT: return 40; case MULTISPLIT: return 38;
      case JOIN: return 41; case MULTIJOIN: return 39; default: return 45; }
  }
  void sig(std::string& o) const override {
    switch (k) {
      case PASS: case MONITOR: o += "MultiPass<1>"; break; case MULTIPASS: o += "MultiPass<" + I(n) + ">"; break;
      case SINK: o += "Sink<" + I(n) + ">"; break; case SPLIT: o += "MultiSplit<1," + I(n) + ">"; break;
      case MULTISPLIT: o += "MultiSplit<" + I(m) + "," + I(n) + ">"; break; case JOIN: o += "MultiJoin<1," + I(n) + ">"; break;
      case MULTIJOIN: o += "MultiJoin<" + I(m) + "," + I(n) + ">"; break; default: o += "Reverse<" + I(n) + ">"; break;
    }
  }
  void lower(Lowering&) const override {}
  HCLONE(Routing)
};

struct Constant : HNode {  // src/audionode.rs:467-523
  std::vector<float> v;
  explicit Constant(std::vector<float> v_) : v(std::move(v_)) {}
  int inputs() const override { return 0; } int outputs() const override { return (int)v.size(); }
  uint64_t id() const override { return 2; }
  void set(const Setting& s) override { if (s.kind == P_VALUE) for (auto& x : v) x = s.v[0]; }
  void sig(std::string& o) const override { o += "Constant<" + I((int)v.size()) + ">"; }
  void lower(Lowering& l) const override { for (float x : v) l.p(x); }
  HCLONE(Constant)
};

// ---------------------------------------------------------------- generators
struct Noise : HNode {  // src/noise.rs:170-234
  bool has_seed = false; uint64_t seed = 0, hash = 0;
  int inputs() const override { return 0; } int outputs() const override { return 1; }
  uint64_t id() const override { return 20; }
  void set(const Setting& s) override { if (s.kind == P_SEED) { has_seed = true; seed = s.seed; } }
  void set_hash(uint64_t h) override { hash = h; }
  void sig(std::string& o) const override { o += "Noise"; }
  void lower(Lowering& l) const override { uint64_t h = has_seed ? seed : hash; l.su((uint32_t)(h ^ (h >> 32))); }
  HCLONE(Noise)
};
struct Sine : HNode {  // src/oscillator.rs:18-102
  uint64_t hash = 0; bool has_phase = false; float initial_phase = 0;
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 21; }
  void set(const Setting& s) override { if (s.kind == P_PHASE) { has_phase = true; initial_phase = s.v[0]; } }
  void set_hash(uint64_t h) override { hash = h; }
  void sig(std::string& o) const override { o += "Sine"; }
  void lower(Lowering& l) const override { l.s(has_phase ? initial_phase : (float)rnd1(hash)); }
  HCLONE(Sine)
};
struct WaveSynth : HNode {  // src/wavetable.rs:244-359
  int kind, nout; uint64_t hash = 0; bool has_phase = false; float initial_phase = 0;
  WaveSynth(int k, int n) : kind(k), nout(n) {}
  int inputs() const override { return 1; } int outputs() const override { return nout; }
  uint64_t id() const override { return 34; }
  void set(const Setting& s) override { if (s.kind == P_PHASE) { has_phase = true; initial_phase = s.v[0]; } }
  void set_hash(uint64_t h) override { hash = h; }
  void sig(std::string& o) const override { o += "WaveSynth<" + I(kind) + "," + I(nout) + ">"; }
  void lower(Lowering& l) const override { l.s(has_phase ? initial_phase : (float)rnd1(hash)); l.su(0u); }
  HCLONE(WaveSynth)
};

struct PhaseSynthN : HNode {  // src/wavetable.rs:361-433
  int kind; explicit PhaseSynthN(int k) : kind(k) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 35; }
  void sig(std::string& o) const override { o += "PhaseSynth<" + I(kind) + ">"; }
  void lower(Lowering& l) const override { l.s(0.0f); l.su(0u); l.su(0u); }   // previous phase, phase_ready, table hint
  HCLONE(PhaseSynthN)
};
struct MixerN : HNode {  // src/pan.rs:95-160
  int m, n; std::vector<float> w;   // w[i * m + j]: weight of input j in output i
  MixerN(int m_, int n_, std::vector<float> w_) : m(m_), n(n_), w(std::move(w_)) {}
  int inputs() const override { return m; } int outputs() const override { return n; }
  uint64_t id() const override { return 84; }
  void sig(std::string& o) const override { o += "Mixer<" + I(m) + "," + I(n) + ">"; }
  void lower(Lowering& l) const override { for (float x : w) l.p(x); }
  HCLONE(MixerN)
};

// ---------------------------------------------------------------- phase oscillators, MLS, impulse, taps
struct PhaseOsc : HNode {  // src/oscillator.rs:440-760
  int kind; uint64_t hash = 0; bool has_phase = false; float initial_phase = 0;
  explicit PhaseOsc(int k) : kind(k) {}
  int inputs() const override { return kind == 3 ? 2 : 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 94 + (uint64_t)kind; }
  void set(const Setting& s) override { if (s.kind == P_PHASE) { has_phase = true; initial_phase = s.v[0]; } }
  void set_hash(uint64_t h) override { hash = h; }
  void sig(std::string& o) const override { o += "PhaseOsc<" + I(kind) + ">"; }
  void lower(Lowering& l) const override { l.s(has_phase ? initial_phase : (float)rnd1(hash)); }
  HCLONE(PhaseOsc)
};
struct DsfN : HNode {  // src/oscillator.rs:114-208
  int nin; float spacing, roughness; uint64_t hash = 0; bool has_phase = false; float initial_phase = 0;
  DsfN(int n, float sp, float r) : nin(n), spacing(sp) { set_roughness(r); }
  void set_roughness(float r) { roughness = fminf(fmaxf(r, 0.0001f), 0.9999f); }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return 55; }
  void set(const Setting& s) override {
    if (s.kind == P_ROUGHNESS) set_roughness(s.v[0]);
    else if (s.kind == P_PHASE) { has_phase = true; initial_phase = s.v[0]; }
  }
  void set_hash(uint64_t h) override { hash = h; }
  void sig(std::string& o) const override { o += "Dsf<" + I(nin) + ">"; }
  void lower(Lowering& l) const override { l.p(roughness); l.p(spacing); l.s(has_phase ? initial_phase : (float)rnd1(hash)); }
  HCLONE(DsfN)
};
const uint32_t kMlsPoly[31] = {
    0b1, 0b11, 0b110, 0b1100, 0b10100, 0b110000, 0b1001000, 0b10111000, 0b100010000, 0b1001000000, 0b10100000000, 0b110010100000,
    0b1101100000000, 0b11000010001000, 0b110000000000000, 0b1101000000001000, 0b10010000000000000, 0b100000010000000000,
    0b1100011000000000000, 0b10010000000000000000, 0b101000000000000000000, 0b1100000000000000000000, 0b10000100000000000000000,
    0b111000010000000000000000, 0b1001000000000000000000000, 0b10000000000000000000100011, 0b100000000000000000000010011,
    0b1001000000000000000000000000, 0b10100000000000000000000000000, 0b100000000000000000000000101001, 0b1001000000000000000000000000000};
struct Mls : HNode {  // src/noise.rs:11-148: unseeded until the first reset (set_hash / .seed())
  uint32_t n, s; bool has_seed = false; uint64_t seed = 0, hash = 0;
  explicit Mls(uint32_t n_) : n(n_), s((1u << n_) - 1u) {}
  int inputs() const override { return 0; } int outputs() const override { return 1; }
  uint64_t id() const override { return 19; }
  void reset() override { uint64_t h = has_seed ? seed : hash; s = 1u + (uint32_t)(h ^ (h >> 32)) % ((1u << n) - 1u); }
  void set(const Setting& st) override { if (st.kind == P_SEED) { has_seed = true; seed = st.seed; } }
  void set_hash(uint64_t h) override { hash = h; reset(); }
  void sig(std::string& o) const override { o += "Mls"; }
  void lower(Lowering& l) const override { l.P.push_back(kMlsPoly[n - 1]); l.P.push_back((1u << n) - 1u); l.P.push_back(n - 1); l.su(s); }
  HCLONE(Mls)
};
struct ImpulseN : HNode {
  int n; explicit ImpulseN(int n_) : n(n_) {}
  int inputs() const override { return 0; } int outputs() const override { return n; }
  uint64_t id() const override { return 81; }
  void sig(std::string& o) const override { o += "Impulse<" + I(n) + ">"; }
  void lower(Lowering& l) const override { l.s(1.0f); }
  HCLONE(ImpulseN)
};
struct TapN : HNode {  // src/delay.rs:141-286 Tap / :379-505 TapLinear
  int ntaps; bool linear; float min_delay, max_delay, sr = 0, lo = 0, hi = 0; uint32_t len = 1;
  TapN(int n, bool lin, float mn, float mx) : ntaps(n), linear(lin), min_delay(mn), max_delay(mx) { set_sample_rate(DEFAULT_SR); }
  int inputs() const override { return ntaps + 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return linear ? 54 : 50; }
  void set_sample_rate(double s) override {
    float f = (float)s;
    if (sr != f) {
      sr = f;
      lo = linear ? min_delay : fmaxf(min_delay, 1.00001f / f);
      hi = linear ? max_delay : fmaxf(max_delay, 1.00001f / f);
      float bl = linear ? ceilf(max_delay * f) + 2.0f : ceilf(max_delay * f) + 3.0f + 8.0f;
      size_t n = (size_t)bl, p2 = 1; while (p2 < n) p2 <<= 1;
      len = (uint32_t)p2;
    }
  }
  void sig(std::string& o) const override { o += "Tap<" + I(ntaps) + "," + I(linear ? 1 : 0) + ">"; }
  void lower(Lowering& l) const override { l.p(lo); l.p(hi); l.U.push_back(len); l.dlen.push_back(len); l.su(0u); }
  HCLONE(TapN)
};

// ---------------------------------------------------------------- SVF (src/svf.rs)
typedef fdsp::SvfCoefs Coefs6;
Coefs6 svf_coefs(int mode, float sr, float cutoff, float q, float gain) {  // src/svf.rs:26-221 (shared host/device code)
  return fdsp::svf_coefs_mode(mode, sr, cutoff, q, gain);
}
struct Svf : HNode {  // FixedSvf (ID 43, :857-1031) and Svf (ID 36, :744-855)
  int mode; bool fixed; float sr, cutoff, q, gain;
  Svf(int m, bool f, float c, float q_, float g) : mode(m), fixed(f), sr((float)DEFAULT_SR), cutoff(c), q(q_), gain(g) {}
  int inputs() const override { return fixed ? 1 : (mode >= 6 ? 4 : 3); } int outputs() const override { return 1; }
  uint64_t id() const override { return fixed ? 43 : 36; }
  void set_sample_rate(double s) override { sr = (float)s; }
  void set(const Setting& s) override {
    if (!fixed) return;
    if (s.kind == P_CENTER) cutoff = s.v[0];
    else if (s.kind == P_CENTER_Q) { cutoff = s.v[0]; q = s.v[1]; }
    else if (s.kind == P_CENTER_Q_GAIN) { cutoff = s.v[0]; q = s.v[1]; gain = s.v[2]; }
  }
  void sig(std::string& o) const override { if (fixed) o += "FixedSvf"; else o += "Svf<" + I(mode) + ">"; }
  void lower(Lowering& l) const override {
    Coefs6 c = svf_coefs(mode, sr, cutoff, q, gain);
    if (fixed) { l.p(c.a1); l.p(c.a2); l.p(c.a3); l.p(c.m0); l.p(c.m1); l.p(c.m2); l.s(0.0f); l.s(0.0f); }
    else { l.s(cutoff); l.s(q); l.s(gain); l.s(sr); l.s(c.a1); l.s(c.a2); l.s(c.a3); l.s(c.m0); l.s(c.m1); l.s(c.m2); l.s(0.0f); l.s(0.0f); }
  }
  HCLONE(Svf)
};

// ---------------------------------------------------------------- prelude64 (F = f64): f64 parameters and state, two words each
struct Sine64 : HNode {  // Sine<f64> src/oscillator.rs:18-102: the initial phase is rnd1(hash) unrounded, or the f32 `.phase()` widened
  uint64_t hash = 0; bool has_phase = false; float initial_phase = 0; double sr = DEFAULT_SR;
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 21; }
  void set_sample_rate(double s) override { sr = s; }
  void set(const Setting& s) override { if (s.kind == P_PHASE) { has_phase = true; initial_phase = s.v[0]; } }
  void set_hash(uint64_t h) override { hash = h; }
  void sig(std::string& o) const override { o += "Sine64"; }
  void lower(Lowering& l) const override { l.p64(1.0 / sr); l.s64(has_phase ? (double)initial_phase : rnd1(hash)); }
  HCLONE(Sine64)
};
SvfCoefs64 svf_coefs64(int mode, double sr, double cutoff, double q, double gain) {  // src/svf.rs:26-221 with F = f64 (shared host/device code)
  switch (mode) {
    case 0: return fdsp::svf_coefs64<0>(sr, cutoff, q, gain); case 1: return fdsp::svf_coefs64<1>(sr, cutoff, q, gain);
    case 2: return fdsp::svf_coefs64<2>(sr, cutoff, q, gain); case 3: return fdsp::svf_coefs64<3>(sr, cutoff, q, gain);
    case 4: return fdsp::svf_coefs64<4>(sr, cutoff, q, gain); case 5: return fdsp::svf_coefs64<5>(sr, cutoff, q, gain);
    case 6: return fdsp::svf_coefs64<6>(sr, cutoff, q, gain); case 7: return fdsp::svf_coefs64<7>(sr, cutoff, q, gain);
    default: return fdsp::svf_coefs64<8>(sr, cutoff, q, gain);
  }
}
struct Svf64 : HNode {  // FixedSvf<f64, M> (ID 43) and Svf<f64, M> (ID 36): the sample rate is convert(sample_rate), settings F::from_f32
  int mode; bool fixed; double sr, cutoff, q, gain;
  Svf64(int m, bool f, float c, float q_, float g) : mode(m), fixed(f), sr(DEFAULT_SR), cutoff(c), q(q_), gain(g) {}
  int inputs() const override { return fixed ? 1 : (mode >= 6 ? 4 : 3); } int outputs() const override { return 1; }
  uint64_t id() const override { return fixed ? 43 : 36; }
  void set_sample_rate(double s) override { sr = s; }
  void set(const Setting& s) override {
    if (!fixed) return;
    if (s.kind == P_CENTER) cutoff = s.v[0];
    else if (s.kind == P_CENTER_Q) { cutoff = s.v[0]; q = s.v[1]; }
    else if (s.kind == P_CENTER_Q_GAIN) { cutoff = s.v[0]; q = s.v[1]; gain = s.v[2]; }
  }
  void sig(std::string& o) const override { if (fixed) o += "FixedSvf64"; else o += "Svf64<" + I(mode) + ">"; }
  void lower(Lowering& l) const override {
    const SvfCoefs64 c = svf_coefs64(mode, sr, cutoff, q, gain);
    if (!fixed) { l.p64(sr); l.s64(cutoff); l.s64(q); l.s64(gain); l.s64(sr); }
    if (fixed) { l.p64(c.a1); l.p64(c.a2); l.p64(c.a3); l.p64(c.m0); l.p64(c.m1); l.p64(c.m2); }
    else { l.s64(c.a1); l.s64(c.a2); l.s64(c.a3); l.s64(c.m0); l.s64(c.m1); l.s64(c.m2); }
    l.s64(0.0); l.s64(0.0);
  }
  HCLONE(Svf64)
};

// Biquad<f64> (ID 15), ButterLowpass<f64, N> (ID 16), Resonator<f64, N> (ID 17): kind 0 arbitrary, 1 butterpass, 2 resonator. The f32
// arguments and settings are widened (F::from_f32); Biquad<f64>::set_sample_rate keeps its coefficients (src/biquad.rs:179-181).
struct Biquad64N : HNode {
  int kind, nin; BqCoefs64 c; double sr, f, q;
  Biquad64N(int kind_, int nin_, const float* k, float f_, float q_) : kind(kind_), nin(nin_), c{0, 0, 0, 0, 0}, sr(DEFAULT_SR), f(f_), q(q_) {
    if (k) { c.a1 = k[0]; c.a2 = k[1]; c.b0 = k[2]; c.b1 = k[3]; c.b2 = k[4]; }
    update();
  }
  void update() { if (kind == 1) c = fdsp::bq_butter_lowpass64(sr, f); else if (kind == 2) c = fdsp::bq_resonator64(sr, f, q); }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return kind == 0 ? 15 : (kind == 1 ? 16 : 17); }
  void set_sample_rate(double s) override { sr = s; update(); }
  void set(const Setting& s) override {
    if (kind == 0 && s.kind == P_BIQUAD) { c.a1 = s.v[0]; c.a2 = s.v[1]; c.b0 = s.v[2]; c.b1 = s.v[3]; c.b2 = s.v[4]; }
    else if (kind == 1 && s.kind == P_CENTER) { f = s.v[0]; update(); }
    else if (kind == 2 && s.kind == P_CENTER_Q) { f = s.v[0]; q = s.v[1]; update(); }
  }
  void sig(std::string& o) const override { if (nin == 1) o += "Biquad64"; else o += "BiquadAudio64<" + I(kind == 1 ? 0 : 1) + ">"; }
  void lower(Lowering& l) const override {
    if (nin == 1) { l.p64(c.a1); l.p64(c.a2); l.p64(c.b0); l.p64(c.b1); l.p64(c.b2); }
    else { l.p64(sr); l.s64(f); l.s64(q); l.s64(sr); l.s64(c.a1); l.s64(c.a2); l.s64(c.b0); l.s64(c.b1); l.s64(c.b2); }
    for (int k = 0; k < 4; k++) l.s64(0.0);
  }
  HCLONE(Biquad64N)
};
// Lowpole / Highpole / Allpole / DCBlock / Pinkpass with F = f64 (src/filter.rs); kinds as mk_onepole
struct OnePole64N : HNode {
  int kind, nin; double param, sr = DEFAULT_SR;
  OnePole64N(int k, float p, int n) : kind(k), nin(n), param(p) {}
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { static const uint64_t ids[5] = {18, 47, 46, 22, 26}; return ids[kind]; }
  void set_sample_rate(double s) override { sr = s; }
  void set(const Setting& s) override {
    if ((kind == 0 || kind == 1 || kind == 3) && s.kind == P_CENTER) param = s.v[0];
    else if (kind == 2 && s.kind == P_DELAY) param = s.v[0];
  }
  void sig(std::string& o) const override { if (kind == 4) o += "Pinkpass64"; else o += "OnePole64<" + I(kind) + "," + I(nin) + ">"; }
  void lower(Lowering& l) const override {
    if (kind == 4) { for (int k = 0; k < 7; k++) l.s64(0.0); return; }
    const double coeff = fdsp::onepole_coeff64(kind, sr, param);
    if (nin == 1) l.p64(coeff); else { l.p64(sr); l.s64(param); l.s64(sr); l.s64(coeff); }
    if (kind != 0) l.s64(0.0);
    l.s64(0.0);
  }
  HCLONE(OnePole64N)
};

struct DeclickN : HNode {  // src/dynamics.rs:245-315
  float duration; explicit DeclickN(float d) : duration(d) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 23; }
  void sig(std::string& o) const override { o += "Declick"; }
  void lower(Lowering& l) const override { l.p(duration); l.s(0.0f); }
  HCLONE(DeclickN)
};
struct ChaosN : HNode {  // Rossler ID 73 / Lorenz ID 74 (src/oscillator.rs:318-438)
  int kind; uint64_t hash = 0;
  explicit ChaosN(int k) : kind(k) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return kind == 0 ? 73 : 74; }
  void set_hash(uint64_t h) override { hash = h; }
  void sig(std::string& o) const override { o += "Chaos<" + I(kind) + ">"; }
  void lower(Lowering& l) const override { const float t = (float)rnd1(hash); l.s(0.0f * (1.0f - t) + 1.0f * t); l.s(1.0f); l.s(1.0f); }
  HCLONE(ChaosN)
};
struct MorphN : HNode {  // src/svf.rs:1034-1111
  Svf filter;
  MorphN(float cutoff, float q) : filter(4, false, cutoff, q, 0.0f) { ctor_ping(); }
  int inputs() const override { return 4; } int outputs() const override { return 1; }
  uint64_t id() const override { return 62; }
  void set_sample_rate(double s) override { filter.set_sample_rate(s); }
  AttoHash ping(bool probe, AttoHash h) override { return filter.ping(probe, h).hash(id()); }
  void sig(std::string& o) const override { o += "Morph"; }
  void lower(Lowering& l) const override { filter.lower(l); }
  HCLONE(MorphN)
};
struct RezN : HNode {  // src/rez.rs
  int nin; float bandpass, cutoff, q, f = 1, fb = 1, sr = (float)DEFAULT_SR;
  RezN(float bp, float c, float qq, int n) : nin(n), bandpass(bp), cutoff(c), q(qq) { update(); }
  void update() { f = 2.0f * m::sinf_(3.14159274101257324f * cutoff / sr); fb = q + q / (1.0f - f); }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return 75; }
  void set_sample_rate(double s) override { sr = (float)s; update(); }
  void set(const Setting& s) override {
    if (s.kind == P_CENTER) { cutoff = s.v[0]; update(); }
    else if (s.kind == P_CENTER_Q) { cutoff = s.v[0]; q = s.v[1]; update(); }
  }
  void sig(std::string& o) const override { o += "Rez<" + I(nin) + ">"; }
  void lower(Lowering& l) const override {
    l.p(bandpass);
    if (nin == 1) { l.p(f); l.p(fb); } else { l.s(cutoff); l.s(q); l.s(sr); l.s(f); l.s(fb); }
    l.s(0.0f); l.s(0.0f);
  }
  HCLONE(RezN)
};

// ---------------------------------------------------------------- biquads (src/biquad.rs, src/biquad_bank.rs)
typedef fdsp::BqCoefs BqCoefs;
BqCoefs bq_butter_lowpass(float sr, float cutoff) { return fdsp::bq_butter_lowpass(sr, cutoff); }   // src/biquad.rs:27-38
BqCoefs bq_resonator(float sr, float center, float q) { return fdsp::bq_resonator(sr, center, q); }  // src/biquad.rs:40-50
struct Biquad : HNode {  // Biquad (ID 15), fixed ButterLowpass (ID 16), fixed Resonator (ID 17)
  int kind;  // 0 arbitrary, 1 butterpass, 2 resonator
  int nin; BqCoefs c; float sr, f, q;
  Biquad(int kind_, int nin_, BqCoefs c_, float f_, float q_) : kind(kind_), nin(nin_), c(c_), sr((float)DEFAULT_SR), f(f_), q(q_) { update(); }
  void update() { if (kind == 1) c = bq_butter_lowpass(sr, f); else if (kind == 2) c = bq_resonator(sr, f, q); }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return kind == 0 ? 15 : (kind == 1 ? 16 : 17); }
  void set_sample_rate(double s) override { sr = (float)s; update(); }
  void set(const Setting& s) override {
    if (kind == 0 && s.kind == P_BIQUAD) { c.a1 = s.v[0]; c.a2 = s.v[1]; c.b0 = s.v[2]; c.b1 = s.v[3]; c.b2 = s.v[4]; }
    else if (kind == 1 && s.kind == P_CENTER) { f = s.v[0]; update(); }
    else if (kind == 2 && s.kind == P_CENTER) { f = s.v[0]; update(); }
    else if (kind == 2 && s.kind == P_CENTER_Q) { f = s.v[0]; q = s.v[1]; update(); }
  }
  void sig(std::string& o) const override { o += nin == 1 ? "Biquad" : (kind == 1 ? "ButterLowpass2" : "Resonator3"); }
  void lower(Lowering& l) const override {
    if (nin == 1) { l.p(c.a1); l.p(c.a2); l.p(c.b0); l.p(c.b1); l.p(c.b2); for (int i = 0; i < 4; i++) l.s(0.0f); return; }
    l.s(f); if (kind == 2) l.s(q);   // audio-rate parameter inputs: the current cutoff / (center, q), the rate and the coefficients are state
    l.s(sr);
    l.s(c.a1); l.s(c.a2); l.s(c.b0); l.s(c.b1); l.s(c.b2); for (int i = 0; i < 4; i++) l.s(0.0f);
  }
  HCLONE(Biquad)
};
struct BiquadBank : HNode {  // src/biquad_bank.rs:9-117
  BqCoefs c[8] = {};
  int inputs() const override { return 8; } int outputs() const override { return 8; }
  uint64_t id() const override { return 98; }
  void set(const Setting& s) override {
    Address d = s.direction();
    if (d.type == 1 && s.kind == P_BIQUAD && d.value < 8) { BqCoefs& k = c[d.value]; k.a1 = s.v[0]; k.a2 = s.v[1]; k.b0 = s.v[2]; k.b1 = s.v[3]; k.b2 = s.v[4]; }
  }
  void sig(std::string& o) const override { o += "BiquadBank"; }
  void lower(Lowering& l) const override {
    for (int k = 0; k < 8; k++) { l.p(c[k].a1); l.p(c[k].a2); l.p(c[k].b0); l.p(c[k].b1); l.p(c[k].b2); }
    for (int k = 0; k < 32; k++) l.s(0.0f);
  }
  HCLONE(BiquadBank)
};

// ---------------------------------------------------------------- Moog (src/moog.rs:11-117)
struct Moog : HNode {
  int nin; float cutoff, q, sr;
  Moog(float c, float q_, int n) : nin(n), cutoff(c), q(q_), sr((float)DEFAULT_SR) {}
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return 60; }
  void set_sample_rate(double s) override { sr = (float)s; }
  void set(const Setting& s) override { if (s.kind == P_CENTER) cutoff = s.v[0]; else if (s.kind == P_CENTER_Q) { cutoff = s.v[0]; q = s.v[1]; } }
  void sig(std::string& o) const override { o += "Moog<" + I(nin) + ">"; }
  void lower(Lowering& l) const override {
    if (nin == 1) {  // :48-57
      float c = 2.0f * cutoff / sr;
      float p = c * (1.8f - 0.8f * c);
      float k = 2.0f * fdsp::m::sinf_(c * 3.14159274101257324f * 0.5f) - 1.0f;
      float t1 = (1.0f - p) * 1.386249f;
      float t2 = 12.0f + t1 * t1;
      float rez = q * (t2 + 6.0f * t1) / (t2 - 6.0f * t1);
      l.p(p); l.p(k); l.p(rez);
    }
    for (int i = 0; i < 8; i++) l.s(0.0f);
  }
  HCLONE(Moog)
};

// ---------------------------------------------------------------- FIR / delays (src/fir.rs, src/delay.rs)
struct Fir : HNode {
  std::vector<float> w;
  explicit Fir(std::vector<float> w_) : w(std::move(w_)) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 52; }
  void sig(std::string& o) const override { o += "Fir<" + I((int)w.size()) + ">"; }
  void lower(Lowering& l) const override { for (float x : w) l.p(x); for (size_t i = 0; i < w.size(); i++) l.s(0.0f); }
  HCLONE(Fir)
};
struct TickN : HNode {
  int n; explicit TickN(int n_) : n(n_) {}
  int inputs() const override { return n; } int outputs() const override { return n; }
  uint64_t id() const override { return 9; }
  void sig(std::string& o) const override { o += "Tick<" + I(n) + ">"; }
  void lower(Lowering& l) const override { for (int i = 0; i < n; i++) l.s(0.0f); }
  HCLONE(TickN)
};
struct Delay : HNode {  // src/delay.rs:67-139: length round(t*sr) + 1, class-uniform
  double time, sr;
  explicit Delay(double t) : time(t), sr(DEFAULT_SR) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 13; }
  void set_sample_rate(double s) override { sr = s; }
  uint32_t len() const { return (uint32_t)((size_t)round(time * sr) + 1); }
  // the length shapes the state, so it is part of the structural signature of the voice class
  void sig(std::string& o) const override { o += "Delay"; }
  void lower(Lowering& l) const override { l.U.push_back(len()); l.dlen.push_back(len()); l.su(0u); }
  HCLONE(Delay)
};
struct AllNest : HNode {  // src/delay.rs:288-377
  int nin; float eta; Kid x;
  AllNest(float c, HNode* x_, int n) : nin(n), eta(c), x(x_) {}
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return 83; }
  void set_sample_rate(double s) override { x->set_sample_rate(s); }
  void set(const Setting& s) override { if (s.kind == P_COEFFICIENT) eta = s.v[0]; }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  void sig(std::string& o) const override { o += "AllNest<" + I(nin) + ","; x->sig(o); o += ">"; }
  void lower(Lowering& l) const override { if (nin == 1) { l.p(eta); l.s(0.0f); } else { l.s(eta); l.s(0.0f); } x->lower(l); }
  HCLONE(AllNest)
};

// ---------------------------------------------------------------- Reverb<F> (src/reverb.rs:139-279) and Var (src/shared.rs:84-131)
struct ReverbN : HNode {
  struct Block { Kid delay, ap0[4], ap1[4], f0, f1; };
  Kid pre[4]; Block block[8]; float a;
  static HNode* schroeder(float coeff, int samples) { return new AllNest(coeff, new Delay((double)(samples - 1) / DEFAULT_SR), 1); }
  ReverbN(double time, double diffusion, HNode* filter) {   // :156-206; the loop filter is cloned into its 16 positions as constructed
    static const int ldelays[32] = {401, 421, 443, 463, 487, 503, 523, 547, 563, 587, 607, 619, 643, 661, 683, 701, 727, 743, 761, 787, 809, 823, 839, 863, 883, 907, 929, 947, 967, 983, 1009, 1021};
    static const int rdelays[32] = {419, 433, 457, 479, 491, 509, 541, 557, 577, 593, 613, 631, 653, 673, 691, 719, 733, 757, 773, 797, 811, 829, 853, 877, 887, 911, 937, 953, 977, 997, 1013, 1033};
    static const int delays[8] = {1087, 1091, 1093, 1097, 1103, 1109, 1117, 1123};
    static const int predelay[4] = {245, 367, 263, 349};
    const float coeff = (float)(0.5 * (1.0 - diffusion) + 0.9 * diffusion);
    for (int i = 0; i < 8; i++) {
      for (int j = 0; j < 4; j++) { block[i].ap0[j] = Kid(schroeder(coeff, ldelays[i + j * 8])); block[i].ap1[j] = Kid(schroeder(coeff, rdelays[i + j * 8])); }
      block[i].delay = Kid(new Delay((double)delays[7 - i] / DEFAULT_SR));
      block[i].f0 = Kid(filter->clone()); block[i].f1 = Kid(filter->clone());
    }
    a = (float)pow(exp((-60.0 / 20.0) * 2.302585092994046), 0.035 / time);   // pow(db_amp(-60.0), 0.035 / time) as f32 (src/math.rs:74-76,294-296)
    for (int i = 0; i < 4; i++) pre[i] = Kid(schroeder(coeff, predelay[i]));
    delete filter;
  }
  int inputs() const override { return 2; } int outputs() const override { return 2; }
  uint64_t id() const override { return 85; }
  template <class Fn> void each(Fn fn) { for (auto& b : block) { for (auto& x : b.ap0) fn(*x); for (auto& x : b.ap1) fn(*x); fn(*b.f0); fn(*b.f1); fn(*b.delay); } }
  void reset() override { each([](HNode& n) { n.reset(); }); }
  void set_sample_rate(double s) override { each([s](HNode& n) { n.set_sample_rate(s); }); }   // the pre-delays keep the default rate (:230-242)
  void sig(std::string& o) const override { o += "Reverb85<"; block[0].f0->sig(o); o += ">"; }
  void lower(Lowering& l) const override {
    l.p(a); l.s(0.0f);
    const uint32_t s0 = (uint32_t)l.S.size(), d0 = (uint32_t)l.dlen.size();
    for (int i = 0; i < 4; i++) pre[i]->lower(l);
    l.keepS.emplace_back(s0, (uint32_t)l.S.size()); l.keepD.emplace_back(d0, (uint32_t)l.dlen.size());   // Reverb::reset leaves `pre` alone (:215-228)
    for (auto& b : block) {
      b.delay->lower(l);
      for (auto& x : b.ap0) x->lower(l);
      b.f0->lower(l);
      for (auto& x : b.ap1) x->lower(l);
      b.f1->lower(l);
    }
  }
  HCLONE(ReverbN)
};
struct FeedbackUnitN : HNode {  // src/feedback.rs:316-481
  Kid x; double delay, sr = 0.0; uint32_t samples = 1, len = 1;
  FeedbackUnitN(double d, HNode* x_) : x(x_), delay(d) { set_sample_rate(DEFAULT_SR); }
  int inputs() const override { return x->inputs(); } int outputs() const override { return x->outputs(); }
  uint64_t id() const override { return 79; }
  void reset() override { x->reset(); }
  void set_sample_rate(double s) override {
    if (sr != s) {
      sr = s;
      x->set_sample_rate(s);
      samples = (uint32_t)fmax(round(delay * s), 1.0);
      len = 1; while (len < samples) len <<= 1;
    }
  }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  void sig(std::string& o) const override { o += "FeedbackUnit<"; x->sig(o); o += ">"; }
  void lower(Lowering& l) const override { l.U.push_back(samples); l.U.push_back(len); l.dlen.push_back(len * (uint32_t)inputs()); l.su(0u); x->lower(l); }
  HCLONE(FeedbackUnitN)
};
struct OnePoleN : HNode {  // src/filter.rs: kind 0 Lowpole, 1 Highpole, 2 Allpole, 3 DCBlock, 4 Pinkpass (F = f32)
  int kind, nin; float param, coeff = 0, sr = (float)DEFAULT_SR;
  OnePoleN(int k, float p, int n) : kind(k), nin(n), param(p) { set_param(p); }
  void set_param(float p) {
    param = p;
    if (kind != 4) coeff = fdsp::onepole_coeff(kind, sr, p);
  }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { static const uint64_t ids[5] = {18, 47, 46, 22, 26}; return ids[kind]; }
  void set_sample_rate(double s) override { sr = (float)s; if (kind != 2 && kind != 4) set_param(param); }
  void set(const Setting& s) override {
    if ((kind == 0 || kind == 1 || kind == 3) && s.kind == P_CENTER) set_param(s.v[0]);
    else if (kind == 2 && s.kind == P_DELAY) set_param(s.v[0]);
  }
  void sig(std::string& o) const override { if (kind == 4) o += "Pinkpass"; else o += "OnePole<" + I(kind) + "," + I(nin) + ">"; }
  void lower(Lowering& l) const override {
    if (kind == 4) { for (int k = 0; k < 7; k++) l.s(0.0f); return; }
    if (nin == 1) l.p(coeff); else { l.s(param); l.s(coeff); if (kind != 2) l.s(sr); }
    if (kind != 0) l.s(0.0f);
    l.s(0.0f);
  }
  HCLONE(OnePoleN)
};
static double halfway_coeff(double samples) {  // src/follow.rs:17-23
  double r0 = log(fmax(1.0, samples)) - 0.861624594696583;
  double r1 = 1.0 / (1.0 + exp(0.0 - r0));
  double r2 = r1 * 1.13228543863477 - 0.1322853859;
  return 1.0 - fmin(0.9999999, r2);
}
struct FollowerN : HNode {  // Follow ID 24 / AFollow ID 29
  bool asym; float atime, rtime, acoeff = 0, rcoeff = 0, sr = 0;
  FollowerN(bool as, float a, float r) : asym(as), atime(a), rtime(r) { set_sample_rate(DEFAULT_SR); }
  void set_time(float a, float r) { atime = a; rtime = r; acoeff = (float)halfway_coeff((double)(atime * sr)); rcoeff = (float)halfway_coeff((double)(rtime * sr)); }
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return asym ? 29 : 24; }
  void set_sample_rate(double s) override { sr = (float)s; set_time(atime, rtime); }
  void set(const Setting& s) override {
    if (!asym && s.kind == P_TIME) set_time(s.v[0], s.v[0]);
    else if (asym && s.kind == P_ATTACK_RELEASE) set_time(s.v[0], s.v[1]);
  }
  void sig(std::string& o) const override { o += "Follower<" + I(asym ? 1 : 0) + ">"; }
  void lower(Lowering& l) const override { l.p(acoeff); l.p(rcoeff); l.s(1.0f); l.s(1.0f); l.s(0.0f); l.s(0.0f); l.s(0.0f); }
  HCLONE(FollowerN)
};
struct LimiterN : HNode {  // src/dynamics.rs:128-243
  int n; double lookahead, sr = DEFAULT_SR; FollowerN follower;
  LimiterN(int n_, float attack, float release) : n(n_), lookahead((double)attack), follower(true, attack * 0.4f, release * 0.4f) {}
  uint32_t length() const { double r = round(sr * lookahead); return r < 1.0 ? 1u : (uint32_t)r; }   // max(1, round(sample_rate * lookahead) as usize)
  int inputs() const override { return n; } int outputs() const override { return n; }
  uint64_t id() const override { return 25; }
  void set_sample_rate(double s) override { sr = s; follower.set_sample_rate(s); }
  void sig(std::string& o) const override { o += "Limiter<" + I(n) + ">"; }
  void lower(Lowering& l) const override {
    const uint32_t L = length(); uint32_t leaf = 1; while (leaf < L) leaf <<= 1;   // usize::next_power_of_two
    l.U.push_back(L); l.U.push_back(leaf);
    l.p(follower.acoeff); l.p(follower.rcoeff);
    l.su(0u); l.su(0u);
    const uint32_t s0 = (uint32_t)l.S.size();
    l.s(1.0f); l.s(1.0f); l.s(0.0f); l.s(0.0f); l.s(0.0f);
    l.keepS.emplace_back(s0, (uint32_t)l.S.size());   // Limiter::reset = set_sample_rate: index, reducer and buffer are cleared, the follower keeps its state (:181-195)
    l.dlen.push_back((uint32_t)n * L + leaf + L + (L & 1u));
  }
  HCLONE(LimiterN)
};
// the first parameter word of a shape kind: Atan(h) multiplies its input by h * PI * 0.5, evaluated left to right in f32 (src/shape.rs:98)
static float shape_word0(int kind, float p0) { return kind == 6 ? p0 * fdsp::PI_F * 0.5f : p0; }
struct ShaperN : HNode {  // src/shape.rs:205-249
  int kind; float p0, p1;
  ShaperN(int k, float a, float b) : kind(k), p0(a), p1(b) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 42; }
  void sig(std::string& o) const override { o += "Shaper<" + I(kind) + ">"; }
  void lower(Lowering& l) const override { l.p(shape_word0(kind, p0)); l.p(p1); }
  HCLONE(ShaperN)
};
// Adaptive<S> (src/shape.rs:156-200): timescale is an f32 field, widened to f64 for the smoothing factor. `reset` is false from
// construction (state 0.0) until the first HNode::reset (state 1e-3).
struct AdaptiveShape {
  int inner; float p0, p1, timescale; bool reset = false;
  float smoothing(double sr) const { return (float)pow(0.5, 1.0 / ((double)timescale * sr)); }
  void lower_params(Lowering& l, double sr) const { l.p(smoothing(sr)); l.p(shape_word0(inner, p0)); l.p(p1); }
  void lower_state(Lowering& l) const { l.s_reset(reset ? 1.0e-3f : 0.0f, 1.0e-3f); }
};
struct ShaperAdaptiveN : HNode {  // Shaper<Adaptive<S>>: Shaper::set_sample_rate reaches the shape (src/shape.rs:226-228)
  AdaptiveShape a; double sr = DEFAULT_SR;
  explicit ShaperAdaptiveN(const AdaptiveShape& s) : a(s) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 42; }
  void reset() override { a.reset = true; }
  void set_sample_rate(double s) override { sr = s; }
  void sig(std::string& o) const override { o += "ShaperAdaptive<" + I(a.inner) + ">"; }
  void lower(Lowering& l) const override { a.lower_params(l, sr); a.lower_state(l); }
  HCLONE(ShaperAdaptiveN)
};
struct NlBiquadN : HNode {  // src/biquad.rs:494-920
  int fb, mode, shape, nin; float p0, p1, sr = (float)DEFAULT_SR, center = 440.0f, q = 1.0f, gain = 1.0f; BqCoefs c;
  NlBiquadN(int fb_, int mode_, int shape_, float p0_, float p1_, int nin_, float ce, float qq, float gg) : fb(fb_), mode(mode_), shape(shape_), nin(nin_), p0(p0_), p1(p1_) {
    update();
    if (nin == 1) { center = ce; q = qq; gain = gg; update(); }
  }
  void update() { c = fdsp::bq_mode(mode, sr, center, q, gain); }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return fb ? (nin == 1 ? 90 : 88) : (nin == 1 ? 91 : 89); }
  void set_sample_rate(double s) override { sr = (float)s; update(); }
  void set(const Setting& s) override {
    if (nin != 1) return;
    if (s.kind == P_CENTER) { center = s.v[0]; update(); }
    else if (s.kind == P_CENTER_Q) { center = s.v[0]; q = s.v[1]; update(); }
    else if (s.kind == P_CENTER_Q_GAIN) { center = s.v[0]; q = s.v[1]; gain = s.v[2]; update(); }
  }
  void sig(std::string& o) const override { o += "NlBiquad<" + I(fb) + "," + I(mode) + "," + I(shape) + "," + I(nin) + ">"; }
  void lower(Lowering& l) const override {
    l.p(shape_word0(shape, p0)); l.p(p1);
    lower_filter(l);
  }
  void lower_filter(Lowering& l) const {
    if (nin == 1) { l.p(c.a1); l.p(c.a2); l.p(c.b0); l.p(c.b1); l.p(c.b2); }
    else { l.s(center); l.s(q); l.s(gain); l.s(sr); l.s(c.a1); l.s(c.a2); l.s(c.b0); l.s(c.b1); l.s(c.b2); }
    l.s(0.0f); l.s(0.0f);
  }
  HCLONE(NlBiquadN)
};
// a nonlinear biquad with an Adaptive shape: one level estimate for FbBiquad, two (shape1, shape2) for DirtyBiquad. The biquads'
// set_sample_rate does not reach the shape (src/biquad.rs:536-539, :745-748): the smoothing stays at Adaptive::new's 44.1 kHz.
struct NlBiquadAdaptiveN : NlBiquadN {
  AdaptiveShape a;
  NlBiquadAdaptiveN(int fb_, int mode_, const AdaptiveShape& s, int nin_, float ce, float qq, float gg) : NlBiquadN(fb_, mode_, s.inner, s.p0, s.p1, nin_, ce, qq, gg), a(s) {}
  void reset() override { a.reset = true; }
  void sig(std::string& o) const override { o += "NlBiquadAdaptive<" + I(fb) + "," + I(mode) + "," + I(a.inner) + "," + I(nin) + ">"; }
  void lower(Lowering& l) const override {
    a.lower_params(l, DEFAULT_SR);
    lower_filter(l);
    a.lower_state(l); if (!fb) a.lower_state(l);
  }
  HCLONE(NlBiquadAdaptiveN)
};
struct ConvolverN : HNode {  // src/convolve.rs:9-59: the impulse response is class-uniform data (voices with the same response share a class)
  std::vector<float> h;
  explicit ConvolverN(std::vector<float> r) : h(std::move(r)) { if (h.empty()) h.push_back(0.0f); }
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 100; }
  void sig(std::string& o) const override { o += "Convolver"; }
  void lower(Lowering& l) const override {
    uint32_t len = 1; while (len < h.size() + 8) len <<= 1;   // the 8-sample block path looks K + 7 samples back
    l.conv_K = (uint32_t)h.size(); l.conv_off = (uint32_t)l.U.size();
    l.U.push_back((uint32_t)h.size()); l.U.push_back(len);
    for (float x : h) l.U.push_back(f2u(x));
    l.extraU += (uint32_t)h.size();
    l.dlen.push_back(len); l.su(0u);
  }
  HCLONE(ConvolverN)
};
struct MeterN : HNode {  // MeterNode, src/dynamics.rs:316-437
  int kind; double timescale, sr = DEFAULT_SR;
  MeterN(int k, double t) : kind(k), timescale(t) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 61; }
  void set_sample_rate(double s) override { sr = s; }
  void sig(std::string& o) const override { o += "MeterNode<" + I(kind) + ">"; }
  void lower(Lowering& l) const override { l.p(kind == 0 ? 0.0f : (float)pow(0.5, 1.0 / (timescale * sr))); l.s(0.0f); }
  HCLONE(MeterN)
};
struct WavePlayerN : HNode {  // src/wave.rs:739-797: the samples of one channel are class-uniform data; the play region is per voice
  std::shared_ptr<const std::vector<float>> wave; uint32_t start, end, loop;   // loop 0xffffffff = none
  WavePlayerN(std::shared_ptr<const std::vector<float>> w, uint32_t s, uint32_t e, uint32_t lp) : wave(std::move(w)), start(s), end(e), loop(lp) {}
  int inputs() const override { return 0; } int outputs() const override { return 1; }
  uint64_t id() const override { return 65; }
  void sig(std::string& o) const override { o += "WavePlayer"; }
  void lower(Lowering& l) const override {
    l.U.push_back((uint32_t)wave->size());
    for (float x : *wave) l.U.push_back(f2u(x));
    l.extraU += (uint32_t)wave->size();
    l.P.push_back(end); l.P.push_back(loop); l.su(start);
  }
  HCLONE(WavePlayerN)
};
struct ResampleN : HNode {  // src/resample.rs:210-300
  Kid x;
  explicit ResampleN(HNode* x_) : x(x_) { AttoHash h = x->ping(true, AttoHash(69)); x->ping(false, h); }   // Resample::new pings the inner node directly (:228-232)
  int inputs() const override { return 1; } int outputs() const override { return x->outputs(); }
  uint64_t id() const override { return 69; }
  void reset() override { x->reset(); }
  void set_sample_rate(double s) override { x->set_sample_rate(s); }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  void sig(std::string& o) const override { o += "Resample<"; x->sig(o); o += ">"; }
  void lower(Lowering& l) const override {
    const double one = 1.0; uint64_t b; memcpy(&b, &one, 8);     // the read position starts at the second sample (:252-256)
    l.su((uint32_t)b); l.su((uint32_t)(b >> 32)); l.su(0u);
    l.dlen.push_back(128u * (uint32_t)x->outputs());
    x->lower(l);
  }
  HCLONE(ResampleN)
};
struct EventN : HNode {  // one Sequencer event as a voice (src/sequencer.rs:55-92 Event, :768-843 process); device: nodes.cuh Event<X>
  Kid x; double start, end, fade_in, fade_out, sr = DEFAULT_SR, time0 = 0.0; int ease; int status0 = 0;
  double loop_arg = 0.0;   // ReplayMode::Loop(t) of the sequencer this event belongs to (0: none)
  double cs = 0.0, ce = 0.0; bool shifted = false;   // current start / end after re-rating shifts (see set_sample_rate); valid when shifted
  EventN(HNode* x_, double s, double e, int ease_, double fi, double fo) : x(x_), start(s), end(e), fade_in(fi), fade_out(fo), ease(ease_) {}
  int inputs() const override { return 0; } int outputs() const override { return x->outputs(); }
  uint64_t id() const override { return 64; }
  void reset() override { x->reset(); }
  static double loop_point_at(double loop_arg, double rate) { return std::max(64.0 * (1.0 / rate), std::round(loop_arg * rate) / rate); }   // Sequencer::reset :644-650
  // Sequencer::set_sample_rate (:685-701) as written: on a CHANGE of rate every ready event is moved to `active`, then reset() runs — which in
  // loop mode moves every active event back by the (new) loop point and leaves it active. An event pushed at the default rate and then re-rated
  // therefore plays its first period shifted: already over (it ends at once, is reset and starts again at its own time) or — when it straddles
  // the loop point — with its tail at the very beginning. Restated so that a re-rated looping bank equals a re-rated reference sequencer.
  void set_sample_rate(double s) override {
    if (loop_arg > 0.0 && s != sr) { if (!shifted) { cs = start; ce = end; shifted = true; } const double lp = loop_point_at(loop_arg, s); cs -= lp; ce -= lp; }
    sr = s; x->set_sample_rate(s);
  }
  void set(const Setting& s) override { x->set(s); }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h); }   // the sequencer never pings its units (AudioUnit::ping default)
  void sig(std::string& o) const override { o += "Event<"; x->sig(o); o += ">"; }
  static void p64(Lowering& l, double v) { uint64_t b; memcpy(&b, &v, 8); l.P.push_back((uint32_t)b); l.P.push_back((uint32_t)(b >> 32)); }
  void lower(Lowering& l) const override {
    p64(l, sr); p64(l, start); p64(l, end); p64(l, fade_in); p64(l, fade_out); l.P.push_back((uint32_t)ease);
    // loop point as Sequencer::reset computes it (:644-650): at least 64 samples, rounded to the nearest sample; +inf when the sequencer does not loop
    const double sd = 1.0 / sr;
    (void)sd;
    p64(l, loop_arg > 0.0 ? loop_point_at(loop_arg, sr) : std::numeric_limits<double>::infinity());
    uint64_t tb; memcpy(&tb, &time0, 8);
    l.su((uint32_t)tb); l.su((uint32_t)(tb >> 32)); l.su((uint32_t)(shifted ? 1 : status0));   // sequencer time at construction (0 unless pushed into a running bank), status ready (re-rated loop event: active)
    const double cs0 = shifted ? cs : start, ce0 = shifted ? ce : end;
    uint64_t sb, eb; memcpy(&sb, &cs0, 8); memcpy(&eb, &ce0, 8);
    l.su((uint32_t)sb); l.su((uint32_t)(sb >> 32)); l.su((uint32_t)eb); l.su((uint32_t)(eb >> 32));   // current start / end (a loop wrap moves them while the event sounds)
    const size_t k = l.shared.size();
    l.sub(x.p.get());
    l.no_writers_since(k, "a sequencer event");
  }
  HCLONE(EventN)
};
struct EnvelopeN : HNode {  // src/envelope.rs:14-183: the closure is evaluated here, at the reference's sample points, when the graph is lowered
  double interval; int nout, t64; EnvelopeFn fn; void* user; double horizon, sr = DEFAULT_SR; uint64_t hash = 0;
  EnvelopeN(double iv, int n, int t64_, EnvelopeFn f, void* u, double hz) : interval(iv), nout(n), t64(t64_), fn(f), user(u), horizon(hz) {}
  int inputs() const override { return 0; } int outputs() const override { return nout; }
  uint64_t id() const override { return 14; }
  void set_sample_rate(double s) override { sr = s; }
  void set_hash(uint64_t h) override { hash = h; }
  void set(const Setting& s) override { if (s.kind == P_INTERVAL) interval = (double)s.v[0]; }   // self.interval = F::from_f32(time)
  void sig(std::string& o) const override { o += "EnvelopeTab<" + I(nout) + "," + I(t64 ? 1 : 0) + ">"; }
  template <class F> void lower_as(Lowering& l) const {
    auto pF = [&](F x) { if (sizeof(F) == 8) { double d = (double)x; uint64_t b; memcpy(&b, &d, 8); l.P.push_back((uint32_t)b); l.P.push_back((uint32_t)(b >> 32)); } else l.p((float)x); };
    auto sF = [&](F x) { if (sizeof(F) == 8) { double d = (double)x; uint64_t b; memcpy(&b, &d, 8); l.su((uint32_t)b); l.su((uint32_t)(b >> 32)); } else l.s((float)x); };
    const F iv = (F)interval, sd = (F)(1.0 / sr);
    std::vector<double> out((size_t)nout);
    std::vector<float> first((size_t)nout), tab;
    fn(0.0, out.data(), user);                                             // reset(): value_0 = value_1 = E(0)
    for (int c = 0; c < nout; c++) first[c] = (float)out[c];
    F t0 = (F)0; uint64_t h = hash; uint32_t K = 0;
    for (;;) {                                                             // next_segment :63-75, the points only
      const F w = (F)rnd1(h);
      const F t1 = t0 + ((F)0.75f * ((F)1 - w) + (F)1.25f * w) * iv;
      fn((double)t1, out.data(), user);
      for (int c = 0; c < nout; c++) tab.push_back((float)out[c]);
      h = h * 6364136223846793005ull + 1ull; t0 = t1; K++;
      if ((double)t1 > horizon || K >= (1u << 22)) break;
    }
    l.U.push_back(K);
    pF(iv); pF(sd);
    for (float x : tab) l.p(x);
    l.extraP += K * (uint32_t)nout;
    sF((F)0); sF((F)0); sF((F)0);
    l.su((uint32_t)hash); l.su((uint32_t)(hash >> 32)); l.su(0u);
    for (int c = 0; c < nout; c++) { l.s(first[c]); l.s(first[c]); l.s(0.0f); l.s(0.0f); }
    l.su(0u); l.su(0u); l.su(0u);
  }
  void lower(Lowering& l) const override { if (t64) lower_as<double>(l); else lower_as<float>(l); }
  HCLONE(EnvelopeN)
};
struct OversampleN : HNode {  // src/oversample.rs:68-245
  Kid x;
  explicit OversampleN(HNode* x_) : x(x_) { x->set_sample_rate(DEFAULT_SR * 2.0); AttoHash h = x->ping(true, AttoHash(51)); x->ping(false, h); }   // Oversampler::new :85-97
  int inputs() const override { return x->inputs(); } int outputs() const override { return x->outputs(); }
  uint64_t id() const override { return 51; }
  void reset() override { x->reset(); }
  void set_sample_rate(double s) override { x->set_sample_rate(s * 2.0); }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  void sig(std::string& o) const override { o += "Oversample<"; x->sig(o); o += ">"; }
  void lower(Lowering& l) const override { l.su(0u); l.su(0u); l.dlen.push_back(128u * (uint32_t)(x->inputs() + x->outputs())); x->lower(l); }
  HCLONE(OversampleN)
};
struct SlotN : HNode {  // src/slot.rs: two instances of one class in the voice (device: nodes.cuh Slot<X>); `newest` is what reset() adopts (:156-172)
  Kid u[2]; int newest = 0, ease = 1; double fade_time = 0.0, sr = DEFAULT_SR;
  explicit SlotN(HNode* x) { u[0] = Kid(x); u[1] = Kid(x->clone()); }
  int inputs() const override { return u[0]->inputs(); } int outputs() const override { return u[0]->outputs(); }
  uint64_t id() const override { return 78; }
  void reset() override { u[0]->reset(); u[1]->reset(); }
  void set_sample_rate(double s) override { sr = s; u[0]->set_sample_rate(s); u[1]->set_sample_rate(s); }
  AttoHash ping(bool, AttoHash h) override { return h.hash(id()); }   // SlotBackend::ping hands its hash to set_hash of the boxed units, which reaches leaves only (:279-291)
  void sig(std::string& o) const override { o += "Slot<"; u[0]->sig(o); o += ">"; }
  static void p64(Lowering& l, double v) { uint64_t b; memcpy(&b, &v, 8); l.P.push_back((uint32_t)b); l.P.push_back((uint32_t)(b >> 32)); }
  void lower(Lowering& l) const override {
    p64(l, sr); p64(l, fade_time); l.P.push_back((uint32_t)ease);
    l.su((uint32_t)newest); l.su(0u); l.su(0u); l.su(0u);   // which, has_next, fade_phase = 0.0
    const size_t k = l.shared.size();
    u[0]->lower(l); u[1]->lower(l);
    l.no_writers_since(k, "a slot");
  }
  HCLONE(SlotN)
};
struct XfadeN : HNode {  // a Net vertex fading from unit x to unit y of any class (Net::crossfade, src/net.rs:480-504); device: nodes.cuh Xfade<X, Y>
  Kid x, y; int ease; float fade_time; double sr = DEFAULT_SR;
  bool done = true;   // what lower() writes: the RESET image has the vertex at its second unit (the fade is an edit of a running net); the bank lowers the live words with done = false
  XfadeN(HNode* x_, HNode* y_, int ease_, float ft) : x(x_), y(y_), ease(ease_), fade_time(ft) {}
  int inputs() const override { return y->inputs(); } int outputs() const override { return y->outputs(); }
  uint64_t id() const override { return y->id(); }
  void reset() override { x->reset(); y->reset(); }
  void set_sample_rate(double s) override { sr = s; x->set_sample_rate(s); y->set_sample_rate(s); }
  void set(const Setting& s) override { y->set(s); }                                   // settings address the vertex's newest unit
  AttoHash ping(bool probe, AttoHash h) override { return y->ping(probe, h); }
  void sig(std::string& o) const override { o += "Xfade<"; x->sig(o); o += ","; y->sig(o); o += ">"; }
  void lower(Lowering& l) const override {
    const float srf = (float)sr;                                                        // the Net's rate is f32 (src/net.rs:132)
    uint32_t w; memcpy(&w, &srf, 4); l.P.push_back(w); memcpy(&w, &fade_time, 4); l.P.push_back(w); l.P.push_back((uint32_t)ease);
    l.su(done ? 1u : 0u); l.su(0u);                                                     // done, fade_phase = 0.0f
    const size_t k = l.shared.size();
    x->lower(l); y->lower(l);
    l.no_writers_since(k, "a crossfade");
  }
  HCLONE(XfadeN)
};
struct VarN : HNode {  // the shared value is control-plane state: it enters as a parameter word and changes through Setting::value
  float value; explicit VarN(float v) : value(v) {}
  int inputs() const override { return 0; } int outputs() const override { return 1; }
  uint64_t id() const override { return 68; }
  void set(const Setting& s) override { if (s.kind == P_VALUE) value = s.v[0]; }
  void sig(std::string& o) const override { o += "Constant<1>"; }   // per block it is a constant (src/shared.rs:118-121)
  void lower(Lowering& l) const override { l.p(value); }
  HCLONE(VarN)
};
// Var over a Shared (src/shared.rs:84-131): the cell's value is a parameter word. The bank rewrites it from the cell before every call
// (Bank::sh_pull), so a set between two calls holds from the first sample of the next call to its end, as a render sees it when nobody
// sets during the call. The device never reaches the cell.
struct VarSharedN : HNode {
  SharedRef s; explicit VarSharedN(SharedCell* c) : s(c) {}
  int inputs() const override { return 0; } int outputs() const override { return 1; }
  uint64_t id() const override { return 68; }
  void sig(std::string& o) const override { o += "Constant<1>"; }
  void lower(Lowering& l) const override { l.shared.push_back({(uint32_t)l.P.size(), s.c, SH_READ}); l.P.push_back(s.c->get()); }
  HCLONE(VarSharedN)
};
// Monitor (src/dynamics.rs:441-520) and Timer (src/shared.rs:203-250) over a Shared: the device leaves the value they would store in a
// state word of their own (nodes.cuh MonitorShared / TimerShared); after a call the bank stores the last writer's word into the cell.
struct VarFnN : HNode {   // VarFn (src/shared.rs:134-200): the closure (closure.cpp) of the cell's value; its word as Var's, then the captures
  SharedRef s; int nout; std::string expr; std::vector<float> caps;
  VarFnN(SharedCell* c, int n, std::string e, std::vector<float> cp) : s(c), nout(n), expr(std::move(e)), caps(std::move(cp)) {}
  int inputs() const override { return 0; } int outputs() const override { return nout; }
  uint64_t id() const override { return 70; }
  void sig(std::string& o) const override { o += "VarFn<" + I(nout) + "," + I((int)caps.size()) + "," + expr + ">"; }
  void lower(Lowering& l) const override {
    l.shared.push_back({(uint32_t)l.P.size(), s.c, SH_READ}); l.P.push_back(s.c->get());
    for (float c : caps) l.p(c);
  }
  HCLONE(VarFnN)
};
struct MonitorSharedN : HNode {
  SharedRef s; int kind; double timescale, sr = DEFAULT_SR;
  MonitorSharedN(SharedCell* c, int k, double t) : s(c), kind(k), timescale(t) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 56; }
  void set_sample_rate(double r) override { sr = r; }
  void sig(std::string& o) const override { o += "MonitorShared<" + I(kind) + ">"; }
  void lower(Lowering& l) const override {   // MeterState: smoothing, state; then the write-back word
    l.p(kind == 0 ? 0.0f : (float)pow(0.5, 1.0 / (timescale * sr))); l.s(0.0f);
    l.shared.push_back({(uint32_t)l.S.size(), s.c, SH_MONITOR}); l.s(0.0f);
  }
  HCLONE(MonitorSharedN)
};
struct TimerN : HNode {
  SharedRef s; double sr = DEFAULT_SR;
  explicit TimerN(SharedCell* c) : s(c) { c->set(0u); }   // Timer::new stores 0.0
  int inputs() const override { return 0; } int outputs() const override { return 0; }
  uint64_t id() const override { return 57; }
  void reset() override { s.c->set(0u); }
  void set_sample_rate(double r) override { sr = r; }
  void sig(std::string& o) const override { o += "TimerShared"; }
  void lower(Lowering& l) const override {   // sample_duration (f64), time (f64), the write-back word
    l.p64(1.0 / sr); l.s64(0.0);
    l.shared.push_back({(uint32_t)l.S.size(), s.c, SH_TIMER}); l.s(0.0f);
  }
  HCLONE(TimerN)
};

// ---------------------------------------------------------------- pan / envelope (src/pan.rs, src/envelope.rs, src/adsr.rs)
struct Panner : HNode {
  int nin; float value;
  Panner(float v, int n) : nin(n), value(v) {}
  int inputs() const override { return nin; } int outputs() const override { return 2; }
  uint64_t id() const override { return 49; }
  void set(const Setting& s) override { if (s.kind == P_PAN) value = s.v[0]; }
  void sig(std::string& o) const override { o += "Panner<" + I(nin) + ">"; }
  void lower(Lowering& l) const override {  // src/pan.rs:14-17
    float lw, rw;
    fdsp::pan_weights(value, lw, rw);
    if (nin == 1) { l.p(lw); l.p(rw); } else { l.s(lw); l.s(rw); }
  }
  HCLONE(Panner)
};
struct AdsrLive : HNode {
  float a, d, s, r, interval; uint64_t hash = 0;
  AdsrLive(float a_, float d_, float s_, float r_) : a(a_), d(d_), s(s_), r(r_), interval((float)0.002) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 53; }
  void set(const Setting& st) override { if (st.kind == P_INTERVAL) interval = st.v[0]; }
  void set_hash(uint64_t h) override { hash = h; }
  void sig(std::string& o) const override { o += "AdsrLive"; }
  void lower(Lowering& l) const override {
    l.p(a); l.p(d); l.p(s); l.p(r); l.p(interval);
    l.su(0u); l.s(0.0f); l.s(-1.0f);              // attacked, attack_start, release_start (adsr.rs:27-33)
    l.s(0.0f); l.s(0.0f); l.s(0.0f);              // t, t_0, t_1
    l.su((uint32_t)hash); l.su((uint32_t)(hash >> 32));  // t_hash
    l.s(0.0f); l.s(0.0f); l.s(0.0f); l.s(0.0f);   // value_0, value_1, value, value_d
    l.su(0u); l.su(0u); l.su(0u);                 // run, run_len, seg_end
  }
  HCLONE(AdsrLive)
};

// ---------------------------------------------------------------- closures of the signal (csrc/host/closure.cpp parses the text)
// The parsed closure is part of the signature; the captured values are per-voice parameter words in Cap<k> order.
// CL_ENVELOPE is Envelope<f32> (src/envelope.rs:14-183) with its closure of time compiled into the voice program: unlike EnvelopeN above
// it stores no sampled values, so it has no horizon and its words do not grow with the length of the render.
struct ClosureN : HNode {
  ClosureKind kind; int nin, nout; std::string expr; std::vector<float> caps;
  float interval = 0.0f; uint64_t hash = 0;   // the envelopes only
  ClosureN(ClosureKind k, int i, int o, std::string e, std::vector<float> c) : kind(k), nin(i), nout(o), expr(std::move(e)), caps(std::move(c)) {}
  bool envelope() const { return kind == CL_ENVELOPE_IN || kind == CL_ENVELOPE; }
  int inputs() const override { return nin; } int outputs() const override { return nout; }
  uint64_t id() const override { return kind == CL_MAP ? 5 : (kind == CL_SHAPE_FN ? 42 : (kind == CL_ENVELOPE ? 14 : 53)); }
  void set(const Setting& s) override { if (envelope() && s.kind == P_INTERVAL) interval = s.v[0]; }   // src/envelope.rs:165-170, :344-348; map and shape_fn have no parameter
  void set_hash(uint64_t h) override { if (envelope()) hash = h; }                                     // envelope.rs:172-175, :350-353
  void sig(std::string& o) const override {
    const std::string nc = I((int)caps.size());
    if (kind == CL_MAP) o += "Map<" + I(nin) + "," + I(nout) + "," + nc + "," + expr + ">";
    else if (kind == CL_SHAPE_FN) o += "ShaperFn<" + nc + "," + expr + ">";
    else if (kind == CL_ENVELOPE) o += "EnvelopeFn<" + I(nout) + "," + nc + "," + expr + ">";
    else o += "EnvelopeInFn<" + I(nin) + "," + I(nout) + "," + nc + "," + expr + ">";
  }
  void lower(Lowering& l) const override {
    for (float c : caps) l.p(c);
    if (!envelope()) return;
    l.p(interval);
    l.s(0.0f); l.s(0.0f); l.s(0.0f);                      // t, t_0, t_1 (reset; the device evaluates E(0) at the first segment)
    l.su((uint32_t)hash); l.su((uint32_t)(hash >> 32));   // t_hash
    for (int k = 0; k < nout; k++) { l.s(0.0f); l.s(0.0f); l.s(0.0f); l.s(0.0f); }   // value_0, value_1, value, value_d
    l.su(0u); l.su(0u); l.su(0u);                         // run, run_len, seg_end
  }
  HCLONE(ClosureN)
};

// ---------------------------------------------------------------- combinators (src/audionode.rs:724-2800)
struct Binary : HNode {
  enum K { PIPE = 6, STACK = 7, BRANCH = 8, BUS = 10, BINOP = 3 } k; int op; Kid x, y;
  Binary(K k_, int op_, HNode* x_, HNode* y_) : k(k_), op(op_), x(x_), y(y_) { ctor_ping(); }
  int inputs() const override { return (k == STACK || k == BINOP) ? x->inputs() + y->inputs() : x->inputs(); }
  int outputs() const override { return k == PIPE ? y->outputs() : ((k == STACK || k == BRANCH) ? x->outputs() + y->outputs() : x->outputs()); }
  uint64_t id() const override { return (uint64_t)k; }
  void reset() override { x->reset(); y->reset(); }
  void set_sample_rate(double s) override { x->set_sample_rate(s); y->set_sample_rate(s); }
  void set(const Setting& s) override {
    Address d = s.direction();
    if (d.type == 1 && d.value == 0) x->set(s.peel()); else if (d.type == 1 && d.value == 1) y->set(s.peel());
  }
  AttoHash ping(bool probe, AttoHash h) override { return y->ping(probe, x->ping(probe, h.hash(id()))); }
  void sig(std::string& o) const override {
    switch (k) { case PIPE: o += "Pipe<"; break; case STACK: o += "Stack<"; break; case BRANCH: o += "Branch<"; break; case BUS: o += "Bus<"; break;
      default: o += "Binop<" + I(op) + ","; }
    x->sig(o); o += ","; y->sig(o); o += ">";
  }
  void lower(Lowering& l) const override { l.sub(x.p.get()); l.sub(y.p.get()); }
  HCLONE(Binary)
};
struct PulseWaveN : HNode {  // src/wavetable.rs:439-491: (saw with phase output | width) >> (saw | phase + width >> saw at that phase) >> difference
  Kid pulse;
  PulseWaveN() {
    HNode* a = new Binary(Binary::STACK, 0, new WaveSynth(0, 2), mk_pass());
    HNode* b = new Binary(Binary::STACK, 0, mk_pass(), new Binary(Binary::PIPE, 0, new Binary(Binary::BINOP, 0, mk_pass(), mk_pass()), new PhaseSynthN(0)));
    pulse = Kid(new Binary(Binary::PIPE, 0, new Binary(Binary::PIPE, 0, a, b), new Binary(Binary::BINOP, 1, mk_pass(), mk_pass())));
  }
  int inputs() const override { return 2; } int outputs() const override { return 1; }
  uint64_t id() const override { return 44; }
  void reset() override { pulse->reset(); }
  void set_sample_rate(double s) override { pulse->set_sample_rate(s); }
  void set(const Setting& s) override {   // pulse.left_mut().left_mut().left_mut().set(setting): straight to the phase-output saw
    Setting t = s; t.address.insert(t.address.begin(), {Address{1, 0}, Address{1, 0}, Address{1, 0}}); pulse->set(t);
  }
  AttoHash ping(bool probe, AttoHash h) override { return pulse->ping(probe, h).hash(id()); }
  void sig(std::string& o) const override { pulse->sig(o); }
  void lower(Lowering& l) const override { pulse->lower(l); }
  HCLONE(PulseWaveN)
};
struct Unary : HNode {
  enum K { UNOP = 4, THRU = 12, FEEDBACK = 11 } k; int kind; float scalar; Kid x;
  Unary(K k_, int kind_, float s, HNode* x_) : k(k_), kind(kind_), scalar(s), x(x_) { ctor_ping(); }
  int inputs() const override { return x->inputs(); }
  int outputs() const override { return k == THRU ? x->inputs() : x->outputs(); }
  uint64_t id() const override { return (uint64_t)k; }
  void reset() override { x->reset(); }
  void set_sample_rate(double s) override { x->set_sample_rate(s); }
  void set(const Setting& s) override { if (k != FEEDBACK) x->set(s); }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  void sig(std::string& o) const override {
    if (k == UNOP) o += "Unop<" + I(kind) + ","; else if (k == THRU) o += "Thru<"; else o += "Feedback<" + I(kind) + ",";
    x->sig(o); o += ">";
  }
  void lower(Lowering& l) const override {
    if (k == UNOP && kind != 0) l.p(scalar);
    if (k == FEEDBACK) for (int i = 0; i < x->inputs(); i++) l.s(0.0f);
    l.sub(x.p.get());
  }
  HCLONE(Unary)
};
struct Feedback2N : HNode {  // src/feedback.rs:180-314
  int had; Kid x, y;
  Feedback2N(HNode* x_, HNode* y_, int h) : had(h), x(x_), y(y_) { ctor_ping(); }
  int inputs() const override { return x->inputs(); } int outputs() const override { return x->outputs(); }
  uint64_t id() const override { return 66; }
  void reset() override { x->reset(); y->reset(); }
  void set_sample_rate(double s) override { x->set_sample_rate(s); y->set_sample_rate(s); }
  AttoHash ping(bool probe, AttoHash h) override { return y->ping(probe, x->ping(probe, h.hash(id()))); }
  void sig(std::string& o) const override { o += "Feedback2<" + I(had) + ","; x->sig(o); o += ","; y->sig(o); o += ">"; }
  void lower(Lowering& l) const override { for (int i = 0; i < x->inputs(); i++) l.s(0.0f); x->lower(l); y->lower(l); }
  HCLONE(Feedback2N)
};
struct Multi : HNode {  // MultiBus 28, MultiStack 30, Reduce 31, MultiBranch 33, Chain 32
  int kind, op; std::vector<Kid> x;
  Multi(int kind_, int op_, int n, HNode** nodes) : kind(kind_), op(op_) { for (int i = 0; i < n; i++) x.emplace_back(nodes[i]); ctor_ping(); }
  int N() const { return (int)x.size(); }
  int inputs() const override { return (kind == 30 || kind == 31) ? x[0]->inputs() * N() : x[0]->inputs(); }
  int outputs() const override { return (kind == 30 || kind == 33) ? x[0]->outputs() * N() : x[0]->outputs(); }
  uint64_t id() const override { return (uint64_t)kind; }
  void reset() override { for (auto& c : x) c->reset(); }
  void set_sample_rate(double s) override { for (auto& c : x) c->set_sample_rate(s); }
  void set(const Setting& s) override { Address d = s.direction(); if (d.type == 1 && d.value < x.size()) x[d.value]->set(s.peel()); }
  AttoHash ping(bool probe, AttoHash h) override { h = h.hash(id()); for (auto& c : x) h = c->ping(probe, h); return h; }
  void sig(std::string& o) const override {
    // all children must share one structure (the reference enforces one type X by construction)
    std::string first; x[0]->sig(first);
    for (auto& c : x) { std::string s; c->sig(s); if (s != first) { o += "Unsupported"; return; } }
    o += "Multi<" + I(kind) + "," + I(op) + "," + I(N()) + "," + first + ">";
  }
  void lower(Lowering& l) const override { for (auto& c : x) l.sub(c.p.get()); }
  HCLONE(Multi)
};

// ---------------------------------------------------------------- System<X, F> (src/system.rs, ID 67): `update(x, dt, f)`
// f is closure text (closure.cpp, CL_UPDATE) whose `x.set(..)` statements are resolved here, once, to the leaves of X they reach, by
// the rules of the combinators' `set` above (Index peels one step into a binary or Multi combinator; Unop and Thru pass the setting on).
// A reached leaf is a target when the device can recompute its coefficients as its host `set` does (nodes.cuh System); a setting the leaf
// ignores is ignored. The values each target was last set to are STATE words of the System (they survive launches, reset and clone,
// and set_sample_rate recomputes the coefficients from them); dt and the captures are parameter words.
struct SystemN : HNode {
  // target kinds (nodes.cuh UpdTarget): 0 FixedSvf, 1 ButterLowpass, 2 Resonator (reached, but it takes no setting), 3 Biquad, 4 Lowpole, 5 Highpole, 6 DCBlock, 7 Constant, 8 Panner<U1>
  struct Target { int kind, mode; std::vector<int> hops; uint32_t off; int nsv; int arg[5]; };
  Kid x; float interval; std::string expr; std::vector<float> caps; std::vector<UpdateSet> sets;
  std::vector<Target> tg; uint32_t nsv = 0; std::string refused;
  std::vector<std::pair<uint32_t, uint32_t>> pending;   // set-value words a set() has just written (relative to the first); a copy starts with none
  SystemN(HNode* x_, float dt, std::string e, std::vector<float> c, std::vector<UpdateSet> st) : x(x_), interval(dt), expr(std::move(e)), caps(std::move(c)), sets(std::move(st)) {
    for (const UpdateSet& u : sets) {
      Setting s; s.kind = u.kind;
      for (uint64_t a : u.address) s.address.push_back({1, a});
      std::vector<int> hops; std::string why;
      HNode* n = reach(s, hops);
      if (!n) continue;                                                    // the address leads nowhere: the reference ignores the setting
      int kind = -1, mode = 0, n_sv = 0;
      if (!classify(n, &kind, &mode, &n_sv)) {
        if (ignores(n, s)) continue;                                       // e.g. a center reaching an oscillator
        if (refused.empty()) {
          std::string g; n->sig(g);
          refused = "update: Setting::" + std::string(setting_name(u.kind)) + " at column " + std::to_string(u.col) + " reaches " + g.substr(0, 80) + " (ID " +
                    std::to_string(n->id()) + "), which an update function cannot set on the device (its targets: FixedSvf, the fixed ButterLowpass / Biquad, "
                    "the fixed one-poles, Constant and Panner<U1>)";
        }
        continue;
      }
      int slots[5];
      if (!accepts(kind, u.kind, slots)) continue;                         // a setting the target ignores
      Target* t = nullptr;
      for (Target& q : tg) if (q.hops == hops) t = &q;
      if (!t) { tg.push_back(Target{kind, mode, hops, nsv, n_sv, {-1, -1, -1, -1, -1}}); t = &tg.back(); nsv += (uint32_t)n_sv; }
      for (int k = 0; k < u.nargs; k++) if (slots[k] >= 0) t->arg[slots[k]] = u.arg + k;   // the last statement to write a value wins
    }
    ctor_ping();   // System::new: the inner node is pinged from AttoHash::new(67) through System::ping (src/system.rs:27-39)
  }
  SystemN(const SystemN& o) : HNode(o), x(o.x), interval(o.interval), expr(o.expr), caps(o.caps), sets(o.sets), tg(o.tg), nsv(o.nsv), refused(o.refused) {}
  // where the setting goes inside X, as the combinators' set() route it; `hops`: the child taken at each step (nodes.cuh UpdAt)
  HNode* reach(Setting s, std::vector<int>& hops) const { return reach_setting(x.p.get(), &s, &hops); }
  static const char* setting_name(int kind) {
    switch (kind) { case P_CENTER: return "center"; case P_CENTER_Q: return "center_q"; case P_CENTER_Q_GAIN: return "center_q_gain";
      case P_VALUE: return "value"; case P_BIQUAD: return "biquad"; default: return "pan"; }
  }
  // a leaf that is not a target but whose set() leaves every word it lowers as it was ignores the setting, as the reference's node does
  static bool ignores(const HNode* n, Setting s) {
    std::unique_ptr<HNode> c(n->clone());
    for (float& v : s.v) v = 1234.5f;
    s.address.clear();
    Lowering a, b;
    c->lower(a); c->set(s); c->lower(b);
    return a.ok && b.ok && a.P == b.P && a.S == b.S && a.U == b.U;
  }
  static bool classify(HNode* n, int* kind, int* mode, int* n_sv) {
    if (Svf* f = dynamic_cast<Svf*>(n)) { if (!f->fixed) return false; *kind = 0; *mode = f->mode; *n_sv = 3; return true; }
    if (Biquad* b = dynamic_cast<Biquad*>(n)) {
      if (b->nin != 1) return false;
      *kind = b->kind == 1 ? 1 : (b->kind == 2 ? 2 : 3); *n_sv = b->kind == 1 ? 1 : (b->kind == 2 ? 0 : 5); return true;
    }
    if (OnePoleN* o = dynamic_cast<OnePoleN*>(n)) {
      if (o->nin != 1 || !(o->kind == 0 || o->kind == 1 || o->kind == 3)) return false;
      *kind = o->kind == 0 ? 4 : (o->kind == 1 ? 5 : 6); *n_sv = 1; return true;
    }
    if (dynamic_cast<Constant*>(n)) { *kind = 7; *n_sv = 1; return true; }
    if (Panner* p = dynamic_cast<Panner*>(n)) { if (p->nin != 1) return false; *kind = 8; *n_sv = 1; return true; }
    return false;
  }
  // the set values a setting of `setting` kind writes on a target of `kind`: slots[k] for its k-th argument (-1: unused); false: ignored
  static bool accepts(int kind, int setting, int* slots) {
    for (int k = 0; k < 5; k++) slots[k] = -1;
    const int n = kind == 0 ? (setting == P_CENTER ? 1 : setting == P_CENTER_Q ? 2 : setting == P_CENTER_Q_GAIN ? 3 : 0)   // FixedSvf::set (src/svf.rs)
                : kind == 1 ? (setting == P_CENTER ? 1 : 0)
                : kind == 2 ? 0                                    // Resonator has no set(): AudioNode's default ignores every setting (src/biquad.rs:340-387)
                : kind == 3 ? (setting == P_BIQUAD ? 5 : 0)
                : kind <= 6 ? (setting == P_CENTER ? 1 : 0)
                : kind == 7 ? (setting == P_VALUE ? 1 : 0)
                : (setting == P_PAN ? 1 : 0);
    for (int k = 0; k < n; k++) slots[k] = k;
    return n > 0;
  }
  HNode* at(const std::vector<int>& hops) const {
    HNode* n = x.p.get();
    for (int h : hops) {
      if (Binary* b = dynamic_cast<Binary*>(n)) n = h == 0 ? b->x.p.get() : b->y.p.get();
      else if (Unary* u = dynamic_cast<Unary*>(n)) n = u->x.p.get();
      else n = static_cast<Multi*>(n)->x[h].p.get();
    }
    return n;
  }
  // the current set values of a target of `kind`, as its host node holds them
  static void values(const HNode* n, int kind, float* v) {
    switch (kind) {
      case 0: { const Svf* f = static_cast<const Svf*>(n); v[0] = f->cutoff; v[1] = f->q; v[2] = f->gain; break; }
      case 1: v[0] = static_cast<const Biquad*>(n)->f; break;
      case 3: { const BqCoefs& c = static_cast<const Biquad*>(n)->c; v[0] = c.a1; v[1] = c.a2; v[2] = c.b0; v[3] = c.b1; v[4] = c.b2; break; }
      case 4: case 5: case 6: v[0] = static_cast<const OnePoleN*>(n)->param; break;
      case 7: v[0] = static_cast<const Constant*>(n)->v[0]; break;
      default: v[0] = static_cast<const Panner*>(n)->value; break;
    }
  }
  void values(const Target& t, float* v) const { values(at(t.hops), t.kind, v); }
  int inputs() const override { return x->inputs(); } int outputs() const override { return x->outputs(); }
  uint64_t id() const override { return 67; }
  void reset() override { x->reset(); }
  void set_sample_rate(double s) override { x->set_sample_rate(s); }
  void set(const Setting& s) override {   // System::set forwards to x; the values it writes on a target are the target's state words too
    x->set(s);
    std::vector<int> hops;
    if (!reach(s, hops)) return;
    int slots[5];
    for (const Target& t : tg)
      if (t.hops == hops && accepts(t.kind, s.kind, slots))
        for (int k = 0; k < 5; k++) if (slots[k] >= 0) pending.emplace_back(t.off + (uint32_t)slots[k], t.off + (uint32_t)slots[k] + 1u);
  }
  AttoHash ping(bool probe, AttoHash h) override { return x->ping(probe, h.hash(id())); }
  void sig(std::string& o) const override {
    o += "System<"; x->sig(o);
    o += "," + I((int)nsv) + "," + I((int)caps.size()) + "," + expr + ",UpdTargets<";
    for (size_t i = 0; i < tg.size(); i++) {
      const Target& t = tg[i];
      o += std::string(i ? "," : "") + "UpdTarget<" + I(t.kind) + "," + I(t.mode) + "," + I((int)t.off);
      for (int k = 0; k < 5; k++) o += "," + I(t.arg[k]);
      o += ",UpdAt<";
      for (size_t j = 0; j < t.hops.size(); j++) o += (j ? "," : "") + I(t.hops[j]);
      o += ">>";
    }
    o += ">>";
  }
  HCLONE(SystemN)
  void lower(Lowering& l) const override {
    if (!refused.empty()) { l.fail(refused); return; }
    l.p(interval); for (float c : caps) l.p(c);
    l.s(0.0f); l.s(0.0f);                                   // time, delta_time
    const uint32_t s0 = (uint32_t)l.S.size();
    for (const Target& t : tg) { float v[5]; values(t, v); for (int k = 0; k < t.nsv; k++) l.s(v[k]); }
    l.keepS.emplace_back(s0, (uint32_t)l.S.size());        // a target's reset leaves its settings alone (e.g. FixedSvf::reset)
    for (auto& w : pending) l.liveS.emplace_back(s0 + w.first, s0 + w.second);
    x->lower(l);
  }
};

// ---------------------------------------------------------------- Net (src/net.rs, src/vertex.rs)
struct NetPort { int type; int node; int port; };  // 0 Zero, 1 Global(port), 2 Local(node, port)
struct HNet : HNode {
  int nin, nout; float sr = (float)DEFAULT_SR;
  struct Vx { Kid unit; std::vector<NetPort> src; };
  std::vector<Vx> vx; std::vector<NetPort> out;
  HNet(int i, int o) : nin(i), nout(o) { out.assign(o, NetPort{0, 0, 0}); }
  int inputs() const override { return nin; } int outputs() const override { return nout; }
  uint64_t id() const override { return 63; }
  void reset() override { for (auto& v : vx) v.unit->reset(); }
  void set_sample_rate(double s) override {  // src/net.rs:1322-1339: the rate is stored as f32
    float f = (float)s;
    if (sr != f) { sr = f; for (auto& v : vx) v.unit->set_sample_rate((double)f); }
  }
  void set(const Setting& s) override { Address d = s.direction(); if (d.type == 2 && d.value < vx.size()) vx[d.value].unit->set(s.peel()); }
  AttoHash ping(bool probe, AttoHash h) override { h = h.hash(id()); for (auto& v : vx) h = v.unit->ping(probe, h); return h; }
  void determine_order_ping() { AttoHash h = ping(true, AttoHash(id())); ping(false, h); }
  // Evaluation order exactly as Net::determine_order_in (src/net.rs:862-916): sinks first through `propagate`, then reversed.
  // Returns false on a cycle (the reference would then read stale buffers; there is no device form for that).
  bool order(std::vector<int>& ord) const {
    const int N = (int)vx.size();
    std::vector<int> unplugged(N, 0); std::vector<char> done(N, 0);
    for (int i = 0; i < N; i++) for (auto& p : vx[i].src) if (p.type == 2) unplugged[p.node]++;
    ord.clear();
    std::vector<int> stack;
    auto propagate = [&](int start) {   // iterative form of the recursive `propagate`
      stack.push_back(start);
      std::vector<size_t> chan(1, 0);
      while (!stack.empty()) {
        const int i = stack.back(); size_t& ch = chan.back();
        if (ch >= vx[i].src.size()) { stack.pop_back(); chan.pop_back(); continue; }
        const NetPort p = vx[i].src[ch++];
        if (p.type == 2 && --unplugged[p.node] == 0) { done[p.node] = 1; ord.push_back(p.node); stack.push_back(p.node); chan.push_back(0); }
      }
    };
    for (int i = 0; i < N; i++) { if (done[i]) continue; if (unplugged[i] == 0) { done[i] = 1; ord.push_back(i); propagate(i); } }
    if ((int)ord.size() < N) return false;
    std::reverse(ord.begin(), ord.end());
    return true;
  }
  // A Net used as a node: one fused `Dag` program (csrc/dsp/nodes.cuh) with the edges encoded in the type expression.
  void sig(std::string& o) const override {
    std::vector<int> ord;
    if (!order(ord) || vx.size() > 65535) { o += "Unsupported"; return; }
    std::vector<int> pos(vx.size(), 0);
    for (size_t k = 0; k < ord.size(); k++) pos[ord[k]] = (int)k;
    auto code = [&](const NetPort& p) { return p.type == 0 ? 0 : (p.type == 1 ? ((1 << 24) | (p.port & 0xff)) : ((2 << 24) | (pos[p.node] << 8) | (p.port & 0xff))); };
    o += "Dag<" + I(nin) + "," + I(nout) + ",VList<";
    for (size_t k = 0; k < ord.size(); k++) {
      const Vx& v = vx[ord[k]];
      if (k) o += ",";
      o += "Vx<"; v.unit->sig(o);
      for (auto& p : v.src) o += "," + I(code(p));
      o += ">";
    }
    o += ">,Outs<";
    for (int c = 0; c < nout; c++) { if (c) o += ","; o += I(code(out[c])); }
    o += ">>";
  }
  void lower(Lowering& l) const override {
    std::vector<int> ord;
    if (!order(ord)) { l.fail("the Net has a cycle (the reference would read stale buffers, src/net.rs:904-911); no device form"); return; }
    if (vx.size() > 65535) { l.fail("Net too large to encode as one program"); return; }
    // The first process()/tick() of a reference Net runs determine_order, which RE-PINGS the Net's own units from a fresh
    // root hash (src/net.rs:839-842): whatever location hash an enclosing graph handed down at construction is replaced.
    // Lowering happens after all construction, i.e. where the reference would be about to process for the first time.
    const_cast<HNet*>(this)->determine_order_ping();
    for (int v : ord) vx[v].unit->lower(l);
  }
  HCLONE(HNet)
};

}  // namespace

HNode* reach_setting(HNode* n, Setting* s, std::vector<int>* hops) {
  for (;;) {
    const Address d = s->direction();
    if (Binary* b = dynamic_cast<Binary*>(n)) {
      if (d.type != 1 || d.value > 1) return nullptr;
      hops->push_back((int)d.value); n = d.value == 0 ? b->x.p.get() : b->y.p.get(); *s = s->peel();
    } else if (Unary* u = dynamic_cast<Unary*>(n)) {
      if (u->k == Unary::FEEDBACK) return nullptr;
      hops->push_back(0); n = u->x.p.get();
    } else if (Multi* m = dynamic_cast<Multi*>(n)) {
      if (d.type != 1 || d.value >= m->x.size()) return nullptr;
      hops->push_back((int)d.value); n = m->x[d.value].p.get(); *s = s->peel();
    } else return n;
  }
}

HNode* mk_net(int inputs, int outputs) { return (inputs < 0 || outputs < 0) ? nullptr : new HNet(inputs, outputs); }
bool is_net(const HNode* n) { return dynamic_cast<const HNet*>(n) != nullptr; }
int net_push(HNode* net, HNode* unit) {
  HNet* n = dynamic_cast<HNet*>(net);
  if (!n || !unit) { delete unit; return -1; }
  unit->set_sample_rate((double)n->sr);
  HNet::Vx v; v.unit = Kid(unit); v.src.assign(unit->inputs(), NetPort{0, 0, 0});
  n->vx.push_back(std::move(v));
  return (int)n->vx.size() - 1;
}
bool net_connect(HNode* net, int s, int sp, int d, int dp) {
  HNet* n = dynamic_cast<HNet*>(net);
  if (!n || s == d || s < 0 || d < 0 || s >= (int)n->vx.size() || d >= (int)n->vx.size() || sp < 0 || sp >= n->vx[s].unit->outputs() || dp < 0 || dp >= n->vx[d].unit->inputs()) return false;
  n->vx[d].src[dp] = NetPort{2, s, sp};
  return true;
}
bool net_connect_input(HNode* net, int gi, int d, int dp) {
  HNet* n = dynamic_cast<HNet*>(net);
  if (!n || gi < 0 || gi >= n->nin || d < 0 || d >= (int)n->vx.size() || dp < 0 || dp >= n->vx[d].unit->inputs()) return false;
  n->vx[d].src[dp] = NetPort{1, 0, gi};
  return true;
}
bool net_connect_output(HNode* net, int s, int sp, int go) {
  HNet* n = dynamic_cast<HNet*>(net);
  if (!n || go < 0 || go >= n->nout || s < 0 || s >= (int)n->vx.size() || sp < 0 || sp >= n->vx[s].unit->outputs()) return false;
  n->out[go] = NetPort{2, s, sp};
  return true;
}
bool net_pass_through(HNode* net, int gi, int go) {
  HNet* n = dynamic_cast<HNet*>(net);
  if (!n || gi < 0 || gi >= n->nin || go < 0 || go >= n->nout) return false;
  n->out[go] = NetPort{1, 0, gi};
  return true;
}
int net_size(const HNode* net) { const HNet* n = dynamic_cast<const HNet*>(net); return n ? (int)n->vx.size() : -1; }

bool net_extract_voices(HNode* net, std::vector<HNode*>& voices, std::string& tree, std::string& err, std::vector<int>* vertex_ids) {
  HNet* n = dynamic_cast<HNet*>(net);
  if (!n) { err = "not a Net"; return false; }
  if (n->nout < 1) { err = "the Net has no outputs"; return false; }
  n->determine_order_ping();
  const int N = (int)n->vx.size();
  std::vector<char> adder(N, 0);
  for (int i = 0; i < N; i++) { std::string s; n->vx[i].unit->sig(s); adder[i] = (s == "Binop<0,MultiPass<1>,MultiPass<1>>"); }
  // per output channel: expand the adder tree iteratively into (leaf sequence, shape string)
  std::vector<int> leaves0; std::string shape0;
  for (int c = 0; c < n->nout; c++) {
    std::vector<int> leaves; std::string shape;
    struct Fr { NetPort p; int stage; };
    std::vector<Fr> st; st.push_back({n->out[c], 0});
    while (!st.empty()) {
      Fr f = st.back(); st.pop_back();
      if (f.stage == 1) { shape.push_back(')'); continue; }
      if (f.p.type != 2) { err = "a Net output is not driven by a vertex (zero/global pass-through outputs are not voice-separable)"; return false; }
      if (adder[f.p.node]) {
        shape.push_back('(');
        st.push_back({NetPort{0, 0, 0}, 1});
        st.push_back({n->vx[f.p.node].src[1], 0});
        st.push_back({n->vx[f.p.node].src[0], 0});
      } else {
        if (f.p.port != c) { err = "voice output ports must map to the same global output channel"; return false; }
        shape.push_back('v');
        leaves.push_back(f.p.node);
      }
    }
    if (c == 0) { leaves0 = leaves; shape0 = shape; }
    else if (leaves != leaves0 || shape != shape0) { err = "the output channels of the Net use different mix trees"; return false; }
  }
  std::vector<char> used(N, 0);
  for (int v : leaves0) {
    if (used[v]) { err = "a voice vertex feeds the mix more than once"; return false; }
    used[v] = 1;
    HNode* u = n->vx[v].unit.p.get();
    if (u->outputs() != n->nout) { err = "every voice vertex must have as many outputs as the Net"; return false; }
    for (int k = 0; k < u->inputs(); k++) if (!(n->vx[v].src[k].type == 1 && n->vx[v].src[k].port == k)) { err = "voice inputs must be the Net's global inputs in order"; return false; }
    if (u->inputs() != 0 && u->inputs() != n->nin) { err = "voice vertices must take all global inputs or none"; return false; }
  }
  for (int i = 0; i < N; i++) if (!used[i] && !adder[i]) { err = "the Net has vertices that are neither voices nor mix adders"; return false; }
  // classify the shape: canonical level-wise adjacent pairing ("pairwise") or left fold ("chain")
  const size_t V = leaves0.size();
  auto pairwise = [&]() { std::vector<std::string> cur(V, "v"); while (cur.size() > 1) { std::vector<std::string> nx; for (size_t i = 0; i + 1 < cur.size(); i += 2) nx.push_back("(" + cur[i] + cur[i + 1] + ")"); if (cur.size() & 1) nx.push_back(cur.back()); cur.swap(nx); } return cur.empty() ? std::string() : cur[0]; };
  auto chain = [&]() { std::string s = "v"; for (size_t i = 1; i < V; i++) s = "(" + s + "v)"; return s; };
  if (V == 1 || shape0 == pairwise()) tree = "pairwise";
  else if (shape0 == chain()) tree = "chain";
  else { err = "the Net's mix tree is neither the level-wise pairwise tree nor a left fold"; return false; }
  for (int v : leaves0) voices.push_back(n->vx[v].unit->clone());
  if (vertex_ids) *vertex_ids = leaves0;   // voice i of the bank is vertex leaves0[i] of the Net (its NodeId in push order)
  return true;
}

namespace {
}  // namespace

// ---------------------------------------------------------------- builders
HNode* mk_constant(int n, const float* v) { return new Constant(std::vector<float>(v, v + n)); }
HNode* mk_pass() { return new Routing(Routing::PASS, 1, 1); }
HNode* mk_monitor() { return new Routing(Routing::MONITOR, 1, 1); }
HNode* mk_multipass(int n) { return new Routing(Routing::MULTIPASS, 1, n); }
HNode* mk_sink(int n) { return new Routing(Routing::SINK, 1, n); }
HNode* mk_split(int n) { return new Routing(Routing::SPLIT, 1, n); }
HNode* mk_multisplit(int m, int n) { return new Routing(Routing::MULTISPLIT, m, n); }
HNode* mk_join(int n) { return new Routing(Routing::JOIN, 1, n); }
HNode* mk_multijoin(int m, int n) { return new Routing(Routing::MULTIJOIN, m, n); }
HNode* mk_reverse(int n) { return new Routing(Routing::REVERSE, 1, n); }
HNode* mk_sine() { return new Sine(); }
HNode* mk_wavesynth(int kind, int outputs) { return (kind < 0 || kind > 5 || outputs < 1 || outputs > 2) ? nullptr : new WaveSynth(kind, outputs); }
HNode* mk_noise() { return new Noise(); }
HNode* mk_fixed_svf(int mode, float cutoff, float q, float gain) { return (mode < 0 || mode > 8) ? nullptr : new Svf(mode, true, cutoff, q, gain); }
HNode* mk_svf(int mode, float cutoff, float q, float gain) { return (mode < 0 || mode > 8) ? nullptr : new Svf(mode, false, cutoff, q, gain); }
HNode* mk_sine64() { return new Sine64(); }
HNode* mk_biquad64(float a1, float a2, float b0, float b1, float b2) { const float k[5] = {a1, a2, b0, b1, b2}; return new Biquad64N(0, 1, k, 0, 0); }
HNode* mk_butterpass64(float cutoff, int nin) { return (nin < 1 || nin > 2) ? nullptr : new Biquad64N(1, nin, nullptr, cutoff, 0); }
HNode* mk_resonator64(float center, float q, int nin) { return (nin != 1 && nin != 3) ? nullptr : new Biquad64N(2, nin, nullptr, center, q); }
HNode* mk_onepole64(int kind, float param, int inputs) {
  if (kind < 0 || kind > 4 || inputs < 1 || inputs > 2 || ((kind == 3 || kind == 4) && inputs != 1)) return nullptr;
  return new OnePole64N(kind, param, inputs);
}
HNode* mk_fixed_svf64(int mode, float cutoff, float q, float gain) { return (mode < 0 || mode > 8) ? nullptr : new Svf64(mode, true, cutoff, q, gain); }
HNode* mk_svf64(int mode, float cutoff, float q, float gain) { return (mode < 0 || mode > 8) ? nullptr : new Svf64(mode, false, cutoff, q, gain); }
HNode* mk_biquad(float a1, float a2, float b0, float b1, float b2) { BqCoefs c{0, 0, 0, 0, 0}; c.a1 = a1; c.a2 = a2; c.b0 = b0; c.b1 = b1; c.b2 = b2; return new Biquad(0, 1, c, 0, 0); }
HNode* mk_biquad_bank() { return new BiquadBank(); }
HNode* mk_butterpass(float cutoff, int nin) { return new Biquad(1, nin, BqCoefs{0, 0, 0, 0, 0}, cutoff, 0); }
HNode* mk_resonator(float center, float q, int nin) { return new Biquad(2, nin, BqCoefs{0, 0, 0, 0, 0}, center, q); }
HNode* mk_moog(float cutoff, float q, int nin) { return (nin != 1 && nin != 3) ? nullptr : new Moog(cutoff, q, nin); }
HNode* mk_fir(int n, const float* w) { return n < 1 ? nullptr : new Fir(std::vector<float>(w, w + n)); }
HNode* mk_tick(int n) { return new TickN(n); }
HNode* mk_delay(double t) { return t < 0.0 ? nullptr : new Delay(t); }
HNode* mk_allnest(float c, HNode* x, int nin) { if (!x || x->inputs() != 1 || x->outputs() != 1) { delete x; return nullptr; } return new AllNest(c, x, nin); }
HNode* mk_phase_osc(int kind) { return (kind < 0 || kind > 3) ? nullptr : new PhaseOsc(kind); }
HNode* mk_reverb3(double time, double diffusion, HNode* filter) {
  if (!filter || filter->inputs() != 1 || filter->outputs() != 1 || !(time > 0.0)) { delete filter; return nullptr; }
  return new ReverbN(time, diffusion, filter);
}
HNode* mk_var(float value) { return new VarN(value); }
HNode* mk_var_shared(SharedCell* s) { return s ? new VarSharedN(s) : nullptr; }
HNode* mk_monitor_shared(SharedCell* s, int kind, double timescale) {
  return (!s || kind < 0 || kind > 2 || (kind > 0 && !(timescale > 0.0))) ? nullptr : new MonitorSharedN(s, kind, timescale);
}
HNode* mk_timer(SharedCell* s) { return s ? new TimerN(s) : nullptr; }
HNode* mk_slot(HNode* x) { return x ? new SlotN(x) : nullptr; }
HNode* mk_oversample(HNode* x) {   // the block path decimates as many channels as X has inputs (:207): more inputs than outputs would index past the outputs
  if (!x || x->outputs() < 1 || x->inputs() > x->outputs()) { delete x; return nullptr; }
  return new OversampleN(x);
}
HNode* mk_envelope(double interval, int outputs, int time_f64, EnvelopeFn f, void* user, double horizon) {
  if (!(interval > 0.0) || outputs < 1 || outputs > 8 || !f || !(horizon >= 0.0) || horizon / interval > 4.0e6) return nullptr;   // assert!(interval > F::zero())
  return new EnvelopeN(time_f64 ? interval : (double)(float)interval, outputs, time_f64, f, user, horizon);
}
// Slot::set (src/slot.rs:64-71) into instance `inst` of a slot voice: false when `n` is not a slot or the unit is of another class
bool slot_arm(HNode* n, HNode* unit, int inst, int ease, double fade_time) {
  SlotN* s = dynamic_cast<SlotN*>(n);
  std::unique_ptr<HNode> keep(unit);
  if (!s || !unit || inst < 0 || inst > 1) return false;
  std::string a, b; unit->sig(a); s->u[0]->sig(b);
  if (a != b || unit->inputs() != s->inputs() || unit->outputs() != s->outputs()) return false;
  unit->set_sample_rate(s->sr);
  s->u[inst] = Kid(keep.release());
  s->newest = inst; s->ease = ease; s->fade_time = fade_time;
  return true;
}
bool is_slot(const HNode* n) { return dynamic_cast<const SlotN*>(n) != nullptr; }
bool slot_fade(const HNode* n, double* fade_time, double* sr) { const SlotN* s = dynamic_cast<const SlotN*>(n); if (!s) return false; *fade_time = s->fade_time; *sr = s->sr; return true; }
HNode* mk_xfade(HNode* x, HNode* y, int ease, float fade_time) {
  if (!x || !y || x->inputs() != y->inputs() || x->outputs() != y->outputs() || ease < 0 || ease > 1 || !(fade_time > 0.0f)) { delete x; delete y; return nullptr; }
  return new XfadeN(x, y, ease, fade_time);
}
// the two units of a crossfading vertex (null when n is not one); `newest` = the unit the vertex is (or will be) left with
bool xfade_set_done(HNode* n, bool done) { XfadeN* q = dynamic_cast<XfadeN*>(n); if (!q) return false; q->done = done; return true; }
bool xfade_fade(const HNode* n, float* fade_time, float* sr) { const XfadeN* q = dynamic_cast<const XfadeN*>(n); if (!q) return false; *fade_time = q->fade_time; *sr = (float)q->sr; return true; }
const HNode* xfade_unit(const HNode* n, int which) { const XfadeN* q = dynamic_cast<const XfadeN*>(n); return q ? (which ? q->y.p.get() : q->x.p.get()) : nullptr; }
HNode* setting_leaf(HNode* voice, Setting* s, bool* ignored) {
  while (EventN* e = dynamic_cast<EventN*>(voice)) voice = e->x.p.get();
  std::vector<int> hops;
  HNode* n = reach_setting(voice, s, &hops);
  *ignored = n == nullptr;
  if (!n || dynamic_cast<SystemN*>(n) || dynamic_cast<HNet*>(n) || dynamic_cast<SlotN*>(n) || dynamic_cast<XfadeN*>(n)) return nullptr;
  return n;
}
bool read_controls(HNode* n, Controls* c) {
  int n_sv = 0;
  *c = Controls();
  if (!SystemN::classify(n, &c->kind, &c->mode, &n_sv) || c->kind == 2) { c->kind = -1; return false; }
  SystemN::values(n, c->kind, c->v);
  if (const Svf* f = dynamic_cast<const Svf*>(n)) c->sr = f->sr;
  else if (const Biquad* b = dynamic_cast<const Biquad*>(n)) c->sr = b->sr;
  else if (const OnePoleN* o = dynamic_cast<const OnePoleN*>(n)) c->sr = o->sr;
  if (const Constant* k = dynamic_cast<const Constant*>(n)) c->nch = (int)k->v.size();
  return true;
}
int controls_taken(int kind, int setting) {
  int slots[5], n = 0;
  if (SystemN::accepts(kind, setting, slots)) for (int k = 0; k < 5; k++) n += slots[k] >= 0;
  return n;
}
Setting controls_setting(const Controls& c) {
  static const int full[9] = {P_CENTER_Q_GAIN, P_CENTER, P_NULL, P_BIQUAD, P_CENTER, P_CENTER, P_CENTER, P_VALUE, P_PAN};
  Setting s;
  s.kind = c.kind >= 0 && c.kind < 9 ? full[c.kind] : P_NULL;
  for (int k = 0; k < 5; k++) s.v[k] = c.v[k];
  return s;
}
bool setting_ignored(const HNode* n, const Setting& s) { return SystemN::ignores(n, s); }
bool event_edit(HNode* n, double end_time, double fade_out) {   // Sequencer::edit on an event (:441-483, no loop: start == original start)
  EventN* e = dynamic_cast<EventN*>(n);
  if (!e) return false;
  e->end = end_time; e->fade_out = fade_out;
  return true;
}
bool event_times(const HNode* n, double* start, double* end) {
  const EventN* e = dynamic_cast<const EventN*>(n);
  if (!e) return false;
  *start = e->start; *end = e->end;
  return true;
}
bool event_loop(const HNode* n, double* loop_seconds) {
  const EventN* e = dynamic_cast<const EventN*>(n);
  if (!e) return false;
  *loop_seconds = e->loop_arg;
  return true;
}
HNode* mk_event_loop(HNode* x, double start, double end, int fade_ease, double fade_in, double fade_out, double loop_seconds) {
  if (!(loop_seconds >= 0.0) || std::isinf(loop_seconds)) { delete x; return nullptr; }
  HNode* n = mk_event(x, start, end, fade_ease, fade_in, fade_out);
  if (n) static_cast<EventN*>(n)->loop_arg = loop_seconds;
  return n;
}
bool event_rerate_resets(const HNode* n, double s) {
  const EventN* e = dynamic_cast<const EventN*>(n);
  return e && s != e->sr && !(e->loop_arg > 0.0);
}
bool event_set_clock(HNode* n, double time) {
  EventN* e = dynamic_cast<EventN*>(n);
  if (!e) return false;
  e->time0 = time;
  return true;
}
HNode* mk_event(HNode* x, double start, double end, int fade_ease, double fade_in, double fade_out) {
  // Sequencer::push asserts fade_in <= duration && fade_out <= duration (:329-330); the device event renders generators
  if (!x || x->inputs() != 0 || x->outputs() < 1 || fade_ease < 0 || fade_ease > 1 || !(fade_in <= end - start) || !(fade_out <= end - start) || !(fade_in >= 0.0) || !(fade_out >= 0.0)) { delete x; return nullptr; }
  return new EventN(x, start, end, fade_ease, fade_in, fade_out);
}
HNode* mk_limiter(int channels, float attack, float release) {
  if (channels < 1 || channels > 8 || !(attack >= 0.0f) || !(release >= 0.0f) || attack > 10.0f) return nullptr;
  return new LimiterN(channels, attack, release);
}
HNode* mk_meter(int kind, double timescale) { return (kind < 0 || kind > 2 || (kind > 0 && !(timescale > 0.0))) ? nullptr : new MeterN(kind, timescale); }
HNode* mk_playwave(const float* samples, uint64_t length, uint64_t start, uint64_t end, int64_t loop_point) {
  if ((!samples && length) || length > (1ull << 28) || end > length || start > 0xfffffffeull || loop_point >= (int64_t)0xffffffffll) return nullptr;   // assert!(end_point <= wave.length())
  auto w = std::make_shared<std::vector<float>>(samples, samples + length);
  return new WavePlayerN(std::move(w), (uint32_t)start, (uint32_t)end, loop_point < 0 ? 0xffffffffu : (uint32_t)loop_point);
}
HNode* mk_resample(HNode* x) {
  if (!x || x->inputs() != 0 || x->outputs() < 1) { delete x; return nullptr; }
  return new ResampleN(x);
}
HNode* mk_phase_synth(int kind) { return (kind < 0 || kind > 5) ? nullptr : new PhaseSynthN(kind); }
HNode* mk_pulse() { return new PulseWaveN(); }
HNode* mk_mixer(int inputs, int outputs, const float* matrix) {
  if (inputs < 1 || outputs < 1 || inputs * outputs > 64 || !matrix) return nullptr;
  return new MixerN(inputs, outputs, std::vector<float>(matrix, matrix + inputs * outputs));
}
HNode* mk_rotate(float angle, float gain) {   // src/prelude.rs:2876-2884 (f32 cos / sin of libm)
  const float c = m::cosf_(angle), s = m::sinf_(angle);
  const float w[4] = {c * gain, -s * gain, s * gain, c * gain};
  return mk_mixer(2, 2, w);
}
HNode* mk_nl_biquad(int fb, int mode, int shape, float p0, float p1, int inputs, float center, float q, float gain) {
  if (mode < 0 || mode > 3 || shape < 0 || shape > 6 || !(inputs == 1 || inputs == (mode == 3 ? 4 : 3))) return nullptr;
  return new NlBiquadN(fb ? 1 : 0, mode, shape, p0, p1, inputs, center, q, gain);
}
static bool adaptive_shape(double timescale, int inner, float p0, float p1, AdaptiveShape* a, std::string& err) {
  if (inner < 0 || inner > 6) { err = "Adaptive: the inner shape must be one of the kinds 0..6 (Clip .. Atan); an Adaptive or a shape_fn inside Adaptive is not supported"; return false; }
  const float ts = (float)timescale;
  if (!(ts > 0.0f) || !std::isfinite(ts)) { err = "Adaptive: the timescale must be a positive finite number of seconds"; return false; }
  a->inner = inner; a->p0 = p0; a->p1 = p1; a->timescale = ts;
  return true;
}
HNode* mk_shaper_adaptive(double timescale, int inner, float p0, float p1, std::string& err) {
  AdaptiveShape a;
  return adaptive_shape(timescale, inner, p0, p1, &a, err) ? new ShaperAdaptiveN(a) : nullptr;
}
HNode* mk_nl_biquad_adaptive(int fb, int mode, double timescale, int inner, float p0, float p1, int inputs, float center, float q, float gain, std::string& err) {
  if (mode < 0 || mode > 3 || !(inputs == 1 || inputs == (mode == 3 ? 4 : 3))) { err = "nl_biquad: mode must be 0..3 and inputs 1 or 3 (4 for the bell)"; return nullptr; }
  AdaptiveShape a;
  if (!adaptive_shape(timescale, inner, p0, p1, &a, err)) return nullptr;
  return new NlBiquadAdaptiveN(fb ? 1 : 0, mode, a, inputs, center, q, gain);
}
HNode* mk_declick(float duration) { return new DeclickN(duration); }
HNode* mk_chaos(int kind) { return (kind < 0 || kind > 1) ? nullptr : new ChaosN(kind); }
HNode* mk_morph(float cutoff, float q) { return new MorphN(cutoff, q); }
HNode* mk_rez(float bandpass, float cutoff, float q, int inputs) { return (inputs != 1 && inputs != 3) ? nullptr : new RezN(bandpass, cutoff, q, inputs); }
HNode* mk_follow(int asym, float attack, float release) { return new FollowerN(asym != 0, attack, asym ? release : attack); }
HNode* mk_shaper(int kind, float p0, float p1) { return (kind < 0 || kind > 6) ? nullptr : new ShaperN(kind, p0, p1); }
HNode* mk_onepole(int kind, float param, int inputs) {
  if (kind < 0 || kind > 4 || inputs < 1 || inputs > 2 || ((kind == 3 || kind == 4) && inputs != 1) || (kind == 2 && inputs == 1 && !(param > 0.0f))) return nullptr;
  return new OnePoleN(kind, param, inputs);
}
HNode* mk_convolve(const float* response, int n) { return (n < 1 || n > (1 << 20) || !response) ? nullptr : new ConvolverN(std::vector<float>(response, response + n)); }
HNode* mk_feedback_unit(double delay, HNode* x) {
  if (!x || x->inputs() != x->outputs() || x->inputs() < 1 || delay < 0.0) { delete x; return nullptr; }
  return new FeedbackUnitN(delay, x);
}
HNode* mk_dsf(int inputs, float spacing, float roughness) { return (inputs < 1 || inputs > 2 || !(spacing > 0.0f)) ? nullptr : new DsfN(inputs, spacing, roughness); }
HNode* mk_mls(int bits) { return (bits < 1 || bits > 31) ? nullptr : new Mls((uint32_t)bits); }
HNode* mk_impulse(int n) { return n < 1 ? nullptr : new ImpulseN(n); }
HNode* mk_tap(int ntaps, int linear, float mn, float mx) { return (ntaps < 1 || mn < 0.0f || mn > mx) ? nullptr : new TapN(ntaps, linear != 0, mn, mx); }
HNode* mk_feedback2(HNode* x, HNode* y, int hadamard) {
  if (!x || !y || x->inputs() != x->outputs() || y->inputs() != y->outputs() || x->inputs() != y->inputs() || (hadamard && (x->inputs() & (x->inputs() - 1)) != 0)) { delete x; delete y; return nullptr; }
  return new Feedback2N(x, y, hadamard ? 1 : 0);
}
HNode* mk_pan(float value) { return new Panner(value, 1); }
HNode* mk_panner() { return new Panner(0.0f, 2); }
HNode* mk_adsr_live(float a, float d, float s, float r) { return new AdsrLive(a, d, s, r); }
// the captured values in Cap<k> order from (name, value) pairs; "" or the reason
static std::string bind_captures(const Closure& c, int ncaptures, const char* const* names, const float* values, std::vector<float>& v) {
  v.assign(c.caps.size(), 0.0f);
  for (size_t k = 0; k < c.caps.size(); k++) {
    int found = -1;
    for (int j = 0; j < ncaptures; j++) if (names[j] && c.caps[k] == names[j]) found = j;
    if (found < 0) return "`" + c.caps[k] + "` is neither a parameter nor a captured value: pass its value as a capture";
    v[k] = values[found];
  }
  for (int j = 0; j < ncaptures; j++) {
    if (!names[j]) return "null capture name";
    bool used = false;
    for (const std::string& n : c.caps) used = used || n == names[j];
    if (!used) return std::string("capture `") + names[j] + "` does not occur in the closure";
    for (int i = 0; i < j; i++) if (names[i] && strcmp(names[i], names[j]) == 0) return std::string("capture `") + names[j] + "` is given twice";
  }
  return "";
}
static HNode* mk_closure_of(SharedCell* cell, int kind, int inputs, int outputs, double interval, const char* text, int ncaptures,
                            const char* const* names, const float* values, std::string& err) {
  const char* what = kind == CL_MAP ? "map" : (kind == CL_SHAPE_FN ? "shape_fn" : (kind == CL_VAR_FN ? "var_fn" : (kind == CL_ENVELOPE ? "envelope" : "envelope_in")));
  auto bad = [&](const std::string& w) -> HNode* { err = std::string(what) + ": " + w; return nullptr; };
  if (kind < CL_MAP || kind > CL_ENVELOPE || (kind == CL_VAR_FN) != (cell != nullptr)) { err = "closure: bad kind"; return nullptr; }
  if (inputs < 0 || inputs > 8 || outputs < 1 || outputs > 8 || (kind == CL_ENVELOPE && inputs != 0)) return bad("arity mismatch: 0-8 inputs and 1-8 outputs");
  if ((kind == CL_ENVELOPE_IN || kind == CL_ENVELOPE) && !(interval > 0.0)) return bad("the interval must be positive");   // Envelope::new / EnvelopeIn::new assert it (src/envelope.rs:59, :230)
  if (ncaptures < 0 || (ncaptures > 0 && (!names || !values))) return bad("bad capture arrays");
  Closure c;
  const std::string e = parse_closure(text, (ClosureKind)kind, inputs, outputs, c);
  if (!e.empty()) return bad(e);
  std::vector<float> v;
  const std::string ce = bind_captures(c, ncaptures, names, values, v);
  if (!ce.empty()) return bad(ce);
  if (kind == CL_VAR_FN) return new VarFnN(cell, outputs, c.expr, std::move(v));
  ClosureN* n = new ClosureN((ClosureKind)kind, kind == CL_SHAPE_FN ? 1 : inputs, kind == CL_SHAPE_FN ? 1 : outputs, c.expr, std::move(v));
  n->interval = (float)interval;   // Envelope<f32> / EnvelopeIn<f32>: F::from_f32 / the f32 interval of prelude32 (src/prelude32.rs:581-724)
  return n;
}
HNode* mk_closure(int kind, int inputs, int outputs, double interval, const char* text, int ncaptures, const char* const* names, const float* values,
                  std::string& err) {
  if (kind == CL_VAR_FN) { err = "closure: bad kind"; return nullptr; }
  return mk_closure_of(nullptr, kind, inputs, outputs, interval, text, ncaptures, names, values, err);
}
HNode* mk_update(HNode* x, float dt, const char* text, int ncaptures, const char* const* names, const float* values, std::string& err) {
  std::unique_ptr<HNode> keep(x);
  if (!x) { err = "update: null node"; return nullptr; }
  if (ncaptures < 0 || (ncaptures > 0 && (!names || !values))) { err = "update: bad capture arrays"; return nullptr; }
  Closure c;
  std::string e = parse_closure(text, CL_UPDATE, 0, 0, c);
  std::vector<float> v;
  if (e.empty()) e = bind_captures(c, ncaptures, names, values, v);
  if (!e.empty()) { err = "update: " + e; return nullptr; }
  return new SystemN(keep.release(), dt, c.expr, std::move(v), c.sets);
}
HNode* mk_var_fn(SharedCell* s, int outputs, const char* text, int ncaptures, const char* const* names, const float* values, std::string& err) {
  if (!s) { err = "var_fn: null Shared"; return nullptr; }
  return mk_closure_of(s, CL_VAR_FN, 0, outputs, 0.0, text, ncaptures, names, values, err);
}

static HNode* bad2(HNode* x, HNode* y) { delete x; delete y; return nullptr; }
HNode* mk_pipe(HNode* x, HNode* y) { if (!x || !y || x->outputs() != y->inputs()) return bad2(x, y); return new Binary(Binary::PIPE, 0, x, y); }
HNode* mk_stack(HNode* x, HNode* y) { if (!x || !y) return bad2(x, y); return new Binary(Binary::STACK, 0, x, y); }
HNode* mk_branch(HNode* x, HNode* y) { if (!x || !y || x->inputs() != y->inputs()) return bad2(x, y); return new Binary(Binary::BRANCH, 0, x, y); }
HNode* mk_bus(HNode* x, HNode* y) { if (!x || !y || x->inputs() != y->inputs() || x->outputs() != y->outputs()) return bad2(x, y); return new Binary(Binary::BUS, 0, x, y); }
HNode* mk_binop(int op, HNode* x, HNode* y) { if (!x || !y || op < 0 || op > 2 || x->outputs() != y->outputs()) return bad2(x, y); return new Binary(Binary::BINOP, op, x, y); }
HNode* mk_thru(HNode* x) { if (!x) return nullptr; return new Unary(Unary::THRU, 0, 0.0f, x); }
HNode* mk_unop(int kind, float scalar, HNode* x) { if (!x || kind < 0 || kind > 3) { delete x; return nullptr; } return new Unary(Unary::UNOP, kind, scalar, x); }
HNode* mk_feedback(HNode* x, int hadamard) {
  if (!x || x->inputs() != x->outputs() || (hadamard && (x->inputs() & (x->inputs() - 1)) != 0)) { delete x; return nullptr; }
  return new Unary(Unary::FEEDBACK, hadamard ? 1 : 0, 0.0f, x);
}
HNode* mk_multi(int kind, int op, int n, HNode** nodes) {
  bool ok = n > 0 && (kind == 28 || kind == 30 || kind == 31 || kind == 33 || kind == 32);
  for (int i = 0; i < n && ok; i++) ok = nodes[i] && nodes[i]->inputs() == nodes[0]->inputs() && nodes[i]->outputs() == nodes[0]->outputs();
  if (ok && kind == 32) ok = nodes[0]->inputs() == nodes[0]->outputs();
  if (!ok) { for (int i = 0; i < n; i++) delete nodes[i]; return nullptr; }
  return new Multi(kind, op, n, nodes);
}

}  // namespace host
}  // namespace fdsp

// The closure parser is part of this translation unit, so that every build of the host graph (the product library, and the CPU
// builds of the host runtime that tests/ make) contains it.
#include "closure.cpp"

// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h). The prelude64 nodes (F = f64) that fundsp_b200 lowers: Sine<f64>
// (src/oscillator.rs:18-102) and the Simper SVF in its fixed and audio-rate forms (src/svf.rs:17-221, 744-1031), restated
// independently of the product's device code (csrc/dsp/nodes.cuh, libm64.cuh) with the oracle's own f64 libm (fo_libm64.h).
// Built with fo_prelude64.cpp as a library of its own; these are fo::Node objects, so fo_nodes.h's combinators take them as children.
#pragma once
#include "fo_nodes.h"
#include "fo_libm64.h"

namespace fo {

// ---- src/oscillator.rs:18-102 Sine<f64>: phase and sample duration in f64, output sin(phase.to_f32() * f32::TAU)
struct Sine64 : Node {
  double phase = 0, sample_duration = 0; uint64_t hash = 0; bool has_phase = false; double initial_phase = 0;
  Sine64() { reset(); set_sample_rate(DEFAULT_SR); }
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 21; }
  void reset() override { phase = has_phase ? initial_phase : rnd1(hash); }
  void set_sample_rate(double sr) override { sample_duration = 1.0 / sr; }
  void tick(const float* in, float* out) override {
    const double p = phase;
    phase += (double)in[0] * sample_duration;
    phase -= std::floor(phase);
    out[0] = m::sinf_((float)p * 6.28318530717958647692f);
  }
  void process(int size, const float* in, float* out) override {
    double p = phase;
    for (int i = 0; i < full_simd_items(size); i++)
      for (int j = 0; j < 8; j++) {
        const float tmp = (float)p;
        p += (double)in[(i << 3) + j] * sample_duration;
        out[(i << 3) + j] = wide_sinf(tmp * 6.28318530717958647692f);
      }
    phase = p - std::floor(p);
    process_remainder(size, in, out);
  }
  void set(const Setting& s) override { if (s.kind == P_PHASE) { has_phase = true; initial_phase = (double)s.v[0]; } }
  void set_hash(uint64_t h) override { hash = h; reset(); }
  FO_CLONE(Sine64)
};

// ---- src/svf.rs:26-221 SvfCoefs<f64>
struct SvfCoefs64 { double a1 = 0, a2 = 0, a3 = 0, m0 = 0, m1 = 0, m2 = 0; };
inline SvfCoefs64 svf_coefs64(int mode, double sr, double cutoff, double q, double gain) {
  const double PI = 3.14159265358979323846;
  SvfCoefs64 c;
  double g = m64::tan(PI * cutoff / sr), k = 1.0 / q;
  const double a = std::sqrt(gain);
  if (mode == 6) k = 1.0 / (q * a);
  else if (mode == 7) g = g / std::sqrt(a);
  else if (mode == 8) g = g * std::sqrt(a);
  c.a1 = 1.0 / (1.0 + g * (g + k)); c.a2 = g * c.a1; c.a3 = g * c.a2;
  static const double M[6][3] = {{0, 0, 1}, {1, 0, -1}, {0, 1, 0}, {1, 0, 0}, {1, 0, -2}, {1, 0, 0}};
  if (mode <= 5) {
    c.m0 = M[mode][0]; c.m1 = (mode == 2) ? 1.0 : (mode == 0 ? 0.0 : (mode == 5 ? -2.0 * k : -k)); c.m2 = M[mode][2];
  } else if (mode == 6) { c.m0 = 1.0; c.m1 = k * (a * a - 1.0); c.m2 = 0.0; }
  else if (mode == 7) { c.m0 = 1.0; c.m1 = k * (a - 1.0); c.m2 = a * a - 1.0; }
  else { c.m0 = a * a; c.m1 = k * (1.0 - a) * a; c.m2 = 1.0 - a * a; }
  return c;
}
// ---- src/svf.rs:744-855 Svf<f64, M> (ID 36) and :857-1031 FixedSvf<f64, M> (ID 43)
struct Svf64 : Node {
  int mode; bool fixed; double sr, cutoff, q, gain; SvfCoefs64 c; double ic1eq = 0, ic2eq = 0;
  Svf64(int mode_, bool fixed_, float cutoff_, float q_, float gain_) : mode(mode_), fixed(fixed_), sr(DEFAULT_SR), cutoff(cutoff_), q(q_), gain(gain_) { update(); }
  void update() { c = svf_coefs64(mode, sr, cutoff, q, gain); }
  int inputs() const override { return fixed ? 1 : (mode >= 6 ? 4 : 3); } int outputs() const override { return 1; }
  uint64_t id() const override { return fixed ? 43 : 36; }
  void reset() override { ic1eq = 0; ic2eq = 0; }
  void set_sample_rate(double s) override { sr = s; update(); }
  void tick(const float* in, float* out) override {
    if (!fixed) {
      const double cu = in[1], qq = in[2], gg = mode >= 6 ? (double)in[3] : gain;
      if (cu != cutoff || qq != q || gg != gain) { cutoff = cu; q = qq; gain = gg; update(); }
    }
    const double v0 = in[0];
    const double v3 = v0 - ic2eq;
    const double v1 = c.a1 * ic1eq + c.a2 * v3;
    const double v2 = ic2eq + c.a2 * ic1eq + c.a3 * v3;
    ic1eq = 2.0 * v1 - ic1eq;
    ic2eq = 2.0 * v2 - ic2eq;
    out[0] = (float)(c.m0 * v0 + c.m1 * v1 + c.m2 * v2);
  }
  void set(const Setting& s) override {
    if (!fixed) return;
    if (s.kind == P_CENTER) { cutoff = s.v[0]; update(); }
    else if (s.kind == P_CENTER_Q) { cutoff = s.v[0]; q = s.v[1]; update(); }
    else if (s.kind == P_CENTER_Q_GAIN) { cutoff = s.v[0]; q = s.v[1]; gain = s.v[2]; update(); }
  }
  FO_CLONE(Svf64)
};

// ---- src/biquad.rs:130-370 Biquad<f64> (ID 15), ButterLowpass<f64, N> (ID 16), Resonator<f64, N> (ID 17); kind 0 / 1 / 2
struct Biquad64 : Node {
  int kind, nin; double sr = DEFAULT_SR, f, q; double a1 = 0, a2 = 0, b0 = 0, b1 = 0, b2 = 0, x1 = 0, x2 = 0, y1 = 0, y2 = 0;
  Biquad64(int kind_, int nin_, const float* k, float f_, float q_) : kind(kind_), nin(nin_), f(f_), q(q_) {
    if (k) { a1 = k[0]; a2 = k[1]; b0 = k[2]; b1 = k[3]; b2 = k[4]; }
    coefs();
  }
  void coefs() {
    const double PI = 3.14159265358979323846;
    if (kind == 1) {                                   // :27-38
      const double t = m64::tan(f * PI / sr), s2 = std::sqrt(2.0);
      const double a0r = 1.0 / (1.0 + s2 * t + t * t);
      a1 = (2.0 * t * t - 2.0) * a0r; a2 = (1.0 - s2 * t + t * t) * a0r; b0 = t * t * a0r; b1 = 2.0 * b0; b2 = b0;
    } else if (kind == 2) {                            // :40-50
      const double r = m64::exp(-PI * f / (q * sr));
      a1 = -2.0 * r * m64::cos(2.0 * PI * f / sr); a2 = r * r; b0 = std::sqrt(1.0 - r * r) * 0.5; b1 = 0.0; b2 = -b0;
    }
  }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return kind == 0 ? 15 : (kind == 1 ? 16 : 17); }
  void reset() override { x1 = x2 = y1 = y2 = 0.0; }
  void set_sample_rate(double s) override { sr = s; coefs(); }
  void tick(const float* in, float* out) override {
    if (nin > 1) {
      const double nf = in[1], nq = kind == 2 ? (double)in[2] : q;
      if (nf != f || nq != q) { f = nf; q = nq; coefs(); }
    }
    const double x0 = in[0];
    const double y0 = b0 * x0 + b1 * x1 + b2 * x2 - a1 * y1 - a2 * y2;
    x2 = x1; x1 = x0; y2 = y1; y1 = y0;
    out[0] = (float)y0;
  }
  void set(const Setting& s) override {
    if (kind == 0 && s.kind == P_BIQUAD) { a1 = s.v[0]; a2 = s.v[1]; b0 = s.v[2]; b1 = s.v[3]; b2 = s.v[4]; }
    else if (kind == 1 && s.kind == P_CENTER) { f = s.v[0]; coefs(); }
    else if (kind == 2 && s.kind == P_CENTER_Q) { f = s.v[0]; q = s.v[1]; coefs(); }
  }
  FO_CLONE(Biquad64)
};

// ---- src/filter.rs with F = f64: kind 0 Lowpole (ID 18), 1 Highpole (47), 2 Allpole (46), 3 DCBlock (22), 4 Pinkpass (26)
struct OnePole64 : Node {
  int kind, nin; double param, sr = DEFAULT_SR, coeff = 0, x1 = 0, y1 = 0, b[7] = {0, 0, 0, 0, 0, 0, 0};
  OnePole64(int kind_, float p, int nin_) : kind(kind_), nin(nin_), param(p) { update(); }
  void update() {
    const double TAU = 2.0 * 3.14159265358979323846;
    switch (kind) {
      case 0: case 1: coeff = m64::exp(-TAU * param / sr); break;
      case 2: coeff = (1.0 - param) / (1.0 + param); break;
      case 3: coeff = 1.0 - TAU / sr * param; break;
      default: break;
    }
  }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { static const uint64_t ids[5] = {18, 47, 46, 22, 26}; return ids[kind]; }
  void reset() override { x1 = y1 = 0.0; for (double& v : b) v = 0.0; }
  void set_sample_rate(double s) override { sr = s; update(); }
  void tick(const float* in, float* out) override {
    const double x = in[0];
    if (kind == 4) {   // :219-238
      b[0] = 0.99886 * b[0] + x * 0.0555179; b[1] = 0.99332 * b[1] + x * 0.0750759; b[2] = 0.96900 * b[2] + x * 0.1538520;
      b[3] = 0.86650 * b[3] + x * 0.3104856; b[4] = 0.55000 * b[4] + x * 0.5329522; b[5] = -0.7616 * b[5] - x * 0.0168980;
      const double o = (b[0] + b[1] + b[2] + b[3] + b[4] + b[5] + b[6] + x * 0.5362) * 0.115830421;
      b[6] = x * 0.115926;
      out[0] = (float)o;
      return;
    }
    if (nin > 1) {
      const double p = in[1];
      if (kind == 2) { param = p; update(); }
      else if (p != param) { param = p; update(); }
    }
    double y;
    switch (kind) {
      case 0: y = (1.0 - coeff) * x + coeff * y1; break;
      case 1: y = coeff * (y1 + x - x1); break;
      case 2: y = coeff * (x - y1) + x1; break;
      default: y = x - x1 + coeff * y1; break;
    }
    x1 = x; y1 = y;
    out[0] = (float)y;
  }
  void set(const Setting& s) override {
    if ((kind == 0 || kind == 1 || kind == 3) && s.kind == P_CENTER) { param = s.v[0]; update(); }
    else if (kind == 2 && s.kind == P_DELAY) { param = s.v[0]; update(); }
  }
  FO_CLONE(OnePole64)
};

}  // namespace fo

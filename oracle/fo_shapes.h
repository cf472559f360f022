// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h). The Atan and Adaptive waveshapes (src/shape.rs:88-104, :156-200) in Shaper
// (ID 42) and in the nonlinear biquads (src/biquad.rs:494-920, IDs 88-91), restated independently of the product's device code
// (csrc/dsp/nodes.cuh, libm.cuh, math.cuh). Built with fo_shapes.cpp as a library of its own; the other shape kinds are those of
// fo_nodes.h's Shaper, reused as they are.
#pragma once
#include "fo_nodes.h"

namespace fo {
namespace m {

// s_atanf.c of FreeBSD msun, as the Rust `libm` crate ports it (src/math/atanf.rs): f32 arithmetic throughout. The table entries are
// given by their bit patterns (the hex values msun lists beside them).
inline float atanf_(float x) {
  static const uint32_t HI[4] = {0x3eed6338u, 0x3f490fdau, 0x3f7b985eu, 0x3fc90fdau};   // atan(0.5), atan(1), atan(1.5), atan(inf): high parts
  static const uint32_t LO[4] = {0x31ac3769u, 0x33222168u, 0x33140fb4u, 0x33a22168u};   // ... and low parts
  static const float AT[5] = {3.3333328366e-01f, -1.9999158382e-01f, 1.4253635705e-01f, -1.0648017377e-01f, 6.1687607318e-02f};
  const uint32_t hx = fbits(x), ix = hx & 0x7fffffffu;
  const bool neg = (hx >> 31) != 0;
  if (ix >= 0x4c800000u) {                                  // |x| >= 2^26
    if (x != x) return x;
    const float z = fromb(HI[3]) + fromb(0x03800000u);       // + 2^-120
    return neg ? -z : z;
  }
  int id = -1;
  if (ix < 0x3ee00000u) {                                   // |x| < 0.4375
    if (ix < 0x39800000u) return x;                         // |x| < 2^-12
  } else {
    x = std::fabs(x);
    if (ix < 0x3f300000u) { id = 0; x = (2.0f * x - 1.0f) / (2.0f + x); }
    else if (ix < 0x3f980000u) { id = 1; x = (x - 1.0f) / (x + 1.0f); }
    else if (ix < 0x401c0000u) { id = 2; x = (x - 1.5f) / (1.0f + 1.5f * x); }
    else { id = 3; x = -1.0f / x; }
  }
  const float z = x * x, w = z * z;
  const float odd = z * (AT[0] + w * (AT[2] + w * AT[4]));
  const float even = w * (AT[1] + w * AT[3]);
  if (id < 0) return x - x * (odd + even);
  const float r = fromb(HI[id]) - ((x * (odd + even) - fromb(LO[id])) - x);
  return neg ? -r : r;
}

}  // namespace m

// `wide` f32x8::atan (Agner Fog's VCL atan_f with Cephes coefficients), one lane. The masks of the vector code become selects:
// small (|v| < sqrt2 - 1): z = |v| / 1; big (|v| > sqrt2 + 1): z = -1 / |v| + pi/2; otherwise z = (|v| - 1) / (|v| + 1) + pi/4.
// polynomial_3 and mul_add without FMA (the convention of wide_sinf); the result takes v's sign bit.
inline float wide_atanf(float v) {
  const float c0 = -3.33329491539E-1f, c1 = 1.99777106478E-1f, c2 = -1.38776856032E-1f, c3 = 8.05374449538E-2f;
  const float sqrt2 = (float)1.41421356237309504880, one = 1.0f;
  const float t = std::fabs(v);
  const bool ge_small = t >= sqrt2 - one;   // cmp_ge(SQRT_2 - ONE)
  const bool le_big = t <= sqrt2 + one;     // cmp_le(SQRT_2 + ONE)
  float s = le_big ? (float)0.785398163397448309616 : (float)1.57079632679489661923;
  if (!ge_small) s = 0.0f;
  float a = le_big ? t : 0.0f;
  if (ge_small) a = a - one;
  float b = le_big ? one : 0.0f;
  if (ge_small) b = b + t;
  const float z = a / b;
  const float zz = z * z;
  const float zz2 = zz * zz;
  const float lo = c1 * zz + c0, hi = c3 * zz + c2;
  float re = hi * zz2 + lo;
  re = re * (zz * z) + z;
  re = re + s;
  return (m::fbits(v) & 0x80000000u) ? -re : re;
}

// One Shape value: a kind of fo_nodes.h's Shaper (0..5), Atan (6), optionally inside Adaptive.
struct XShape {
  int kind; float p0, p1;
  bool adaptive = false; float timescale = 0.0f, smoothing = 0.0f, state = 0.0f;
  XShape(int k, float a, float b) : kind(k), p0(a), p1(b) {}
  static XShape make_adaptive(float timescale, int k, float a, float b) {   // Adaptive::new: state 0, smoothing at DEFAULT_SR
    XShape s(k, a, b);
    s.adaptive = true; s.timescale = timescale; s.set_sample_rate(DEFAULT_SR);
    return s;
  }
  float inner(float x) const {   // Shape::shape of the plain kind
    if (kind == 6) return m::atanf_(x * (p0 * 3.14159265358979323846f * 0.5f)) * (2.0f / 3.14159265358979323846f);
    return Shaper(kind, p0, p1).shape(x);
  }
  float shape(float x) {
    if (!adaptive) return inner(x);
    state = smoothing * state + (1.0f - smoothing) * (1.0e-6f + x * x);
    return inner(x / std::sqrt(state));
  }
  float simd(float x) {           // Shape::simd, one lane
    if (adaptive) return shape(x);   // the trait default: lane by lane through `shape`
    if (kind == 6) return wide_atanf(x * (p0 * 3.14159265358979323846f * 0.5f)) * (2.0f / 3.14159265358979323846f);
    return Shaper(kind, p0, p1).simd(x);
  }
  void reset() { if (adaptive) state = 1.0e-3f; }
  void set_sample_rate(double sr) { if (adaptive) smoothing = (float)std::pow(0.5, 1.0 / ((double)timescale * sr)); }
};

// Shaper<S> (ID 42) for the shapes above
struct XShaper : Node {
  XShape s;
  explicit XShaper(const XShape& s_) : s(s_) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 42; }
  void reset() override { s.reset(); }
  void set_sample_rate(double sr) override { s.set_sample_rate(sr); }
  void tick(const float* in, float* out) override { out[0] = s.shape(in[0]); }
  void process(int size, const float* in, float* out) override {   // src/shape.rs:235-240
    for (int i = 0; i < (size & ~7); i++) out[i] = s.simd(in[i]);
    process_remainder(size, in, out);
  }
  FO_CLONE(XShaper)
};

// FbBiquad / DirtyBiquad with one of the shapes above; Shape::shape on every path. DirtyBiquad clones its shape (shape1, shape2).
// Neither reset nor set_sample_rate of the biquad is the shape's: reset() resets the shapes, set_sample_rate leaves them alone.
struct XNlBiquad : Node {
  bool fb; int mode, nin; XShape shape1, shape2; BiquadCoefs c;
  float sr = (float)DEFAULT_SR, center = 440.0f, q = 1.0f, gain = 1.0f, s1 = 0.0f, s2 = 0.0f;
  XNlBiquad(bool fb_, int mode_, const XShape& sh, int nin_, float center_, float q_, float gain_) : fb(fb_), mode(mode_), nin(nin_), shape1(sh), shape2(sh) {
    update();
    if (nin == 1) { center = center_; q = q_; gain = gain_; update(); }
  }
  void update() {
    if (mode == 0) c = biquad_resonator(sr, center, q);
    else if (mode == 1) c = biquad_lowpass(sr, center, q);
    else if (mode == 2) c = biquad_highpass(sr, center, q);
    else c = biquad_bell(sr, center, q, gain);
  }
  int inputs() const override { return nin; } int outputs() const override { return 1; }
  uint64_t id() const override { return fb ? (nin == 1 ? 90 : 88) : (nin == 1 ? 91 : 89); }
  void reset() override { s1 = 0.0f; s2 = 0.0f; shape1.reset(); shape2.reset(); }
  void set_sample_rate(double s) override { sr = (float)s; update(); }
  void tick(const float* in, float* out) override {
    if (nin > 1) {
      const float dc = in[1] - center, dq = in[2] - q;
      const float dg = nin == 4 ? in[3] - gain : 0.0f;
      const float test = nin == 4 ? dc * dc + dq * dq + dg * dg : dc * dc + dq * dq;
      if (test != 0.0f) { center = in[1]; q = in[2]; if (nin == 4) gain = in[3]; update(); }
    }
    const float x0 = in[0], y0 = c.b0 * x0 + s1;
    if (fb) {
      const float f = shape1.shape(y0);
      s1 = s2 + c.b1 * x0 - f * c.a1;
      s2 = c.b2 * x0 - f * c.a2;
    } else {
      s1 = shape1.shape(s2 + c.b1 * x0 - y0 * c.a1);
      s2 = shape2.shape(c.b2 * x0 - y0 * c.a2);
    }
    out[0] = y0;
  }
  void set(const Setting& st) override {
    if (nin != 1) return;
    if (st.kind == P_CENTER) { center = st.v[0]; update(); }
    else if (st.kind == P_CENTER_Q) { center = st.v[0]; q = st.v[1]; update(); }
    else if (st.kind == P_CENTER_Q_GAIN) { center = st.v[0]; q = st.v[1]; gain = st.v[2]; update(); }
  }
  FO_CLONE(XNlBiquad)
};

}  // namespace fo

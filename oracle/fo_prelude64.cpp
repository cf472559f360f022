// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h). C ABI of the prelude64 nodes of fo_prelude64.h and of the oracle's f64 libm,
// linked into oracle/_build/libfundsp_oracle.so with fundsp_oracle.cpp (oracle/Makefile); the combinators there take them as children.
#include "fo_prelude64.h"

using namespace fo;

#define API extern "C" __attribute__((visibility("default")))

API double fo64_sin(double x) { return m64::sin(x); }
API double fo64_cos(double x) { return m64::cos(x); }
API double fo64_tan(double x) { return m64::tan(x); }
API double fo64_exp(double x) { return m64::exp(x); }
// the two argument reductions of the trig functions, for finite x: n with x = n pi/2 + y[0] + y[1] (the large one returns n mod 8)
API int fo64_rem_pio2_medium(double x, double* y) { return m64::rem_pio2(x, y); }
API int fo64_rem_pio2_large(double x, double* y) { return m64::rem_pio2_big(x, y); }
// fn = 0 sin, 1 cos, 2 tan, 3 exp over n arguments
API void fo64_eval(int fn, const double* x, double* out, int64_t n) {
  for (int64_t i = 0; i < n; i++) out[i] = fn == 0 ? m64::sin(x[i]) : fn == 1 ? m64::cos(x[i]) : fn == 2 ? m64::tan(x[i]) : m64::exp(x[i]);
}
API Node* fo_sine_f64() { return new Sine64(); }
API Node* fo_fixed_svf_f64(int mode, float cutoff, float q, float gain) { return (mode < 0 || mode > 8) ? nullptr : new Svf64(mode, true, cutoff, q, gain); }
API Node* fo_svf_f64(int mode, float cutoff, float q, float gain) { return (mode < 0 || mode > 8) ? nullptr : new Svf64(mode, false, cutoff, q, gain); }
API Node* fo_biquad_f64(float a1, float a2, float b0, float b1, float b2) { const float k[5] = {a1, a2, b0, b1, b2}; return new Biquad64(0, 1, k, 0, 0); }
API Node* fo_butterpass_f64(float f, int nin) { return (nin < 1 || nin > 2) ? nullptr : new Biquad64(1, nin, nullptr, f, 0); }
API Node* fo_resonator_f64(float f, float q, int nin) { return (nin != 1 && nin != 3) ? nullptr : new Biquad64(2, nin, nullptr, f, q); }
API Node* fo_onepole_f64(int kind, float p, int nin) {
  return (kind < 0 || kind > 4 || nin < 1 || nin > 2 || (kind >= 3 && nin != 1)) ? nullptr : new OnePole64(kind, p, nin);
}
// the phase of a Sine<f64> whose hash is `hash` after set_sample_rate(sr) and n ticks at frequency f (a pin on the unrounded phase)
API double fo_sine_f64_phase_after(uint64_t hash, double sr, float f, int n) {
  Sine64 s; s.set_hash(hash); s.set_sample_rate(sr);
  float y;
  for (int i = 0; i < n; i++) s.tick(&f, &y);
  return s.phase;
}

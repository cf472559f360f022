// fundsp_b200.hpp — header-only C++ host mirror of the reference's graph notation over the C ABI (fundsp_b200.h).
//
// The reference is Rust; where no Rust toolchain exists the host side above the C ABI is C++. This header gives C++
// callers the same surface the reference gives Rust callers for this path:
//   * `An` wraps a graph node like `An<X>` (src/combinator.rs:178) and overloads the same operators with the same
//     meaning and precedence: `>>` Pipe, `|` Stack, `&` Bus, `^` Branch, `+ - *` Binop (or Unop with a float), unary `-`,
//     and `!` Thru (src/combinator.rs:289-488); `.phase()` / `.seed()` as in src/combinator.rs:263-276.
//   * the opcode constructors keep the prelude's names and argument order (src/prelude.rs): sine_hz, saw_hz, white,
//     lowpass_hz, moog_hz, delay, pan, reverb-style building blocks, ...
//   * `Bank` is the AudioUnit: process() == AudioUnit::process (src/audiounit.rs:45), render() == the Wave::render loop.
// Nodes are move-only like Rust values: combining consumes the operands (use clone() to reuse a sub-graph).
#pragma once
#include <cmath>
#include <cstdint>
#include <initializer_list>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "fundsp_b200.h"

namespace fundsp_b200 {

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
inline void check(int rc) { if (rc != FDSP_OK) throw Error(rc, fdsp_last_error()); }

class An {
  fdsp_node* h_;
  static fdsp_node* need(fdsp_node* h) { if (!h) throw Error(FDSP_ERR_ARITY, fdsp_last_error()); return h; }

 public:
  explicit An(fdsp_node* h) : h_(need(h)) {}
  An(An&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
  An& operator=(An&& o) noexcept { if (this != &o) { fdsp_node_free(h_); h_ = o.h_; o.h_ = nullptr; } return *this; }
  An(const An&) = delete;
  An& operator=(const An&) = delete;
  ~An() { fdsp_node_free(h_); }
  An clone() const { return An(fdsp_node_clone(h_)); }
  fdsp_node* release() { fdsp_node* h = h_; h_ = nullptr; return h; }
  const fdsp_node* get() const { return h_; }
  int inputs() const { return fdsp_node_inputs(h_); }
  int outputs() const { return fdsp_node_outputs(h_); }
  An phase(float p) && { check(fdsp_node_phase(h_, p)); return std::move(*this); }
  An seed(uint64_t s) && { check(fdsp_node_seed(h_, s)); return std::move(*this); }
  std::string signature() const { std::string s(1 << 16, '\0'); int n = fdsp_node_signature(h_, &s[0], (int)s.size()); s.resize(n > 0 ? n : 0); return s; }
};

// ---- operators (src/combinator.rs:289-488)
inline An operator>>(An x, An y) { return An(fdsp_pipe(x.release(), y.release())); }
inline An operator|(An x, An y) { return An(fdsp_stack(x.release(), y.release())); }
inline An operator&(An x, An y) { return An(fdsp_bus(x.release(), y.release())); }
inline An operator^(An x, An y) { return An(fdsp_branch(x.release(), y.release())); }
inline An operator!(An x) { return An(fdsp_thru(x.release())); }
inline An operator-(An x) { return An(fdsp_unop(0, 0.0f, x.release())); }
inline An operator+(An x, An y) { return An(fdsp_binop(0, x.release(), y.release())); }
inline An operator-(An x, An y) { return An(fdsp_binop(1, x.release(), y.release())); }
inline An operator*(An x, An y) { return An(fdsp_binop(2, x.release(), y.release())); }
inline An operator+(An x, float y) { return An(fdsp_unop(1, y, x.release())); }
inline An operator+(float y, An x) { return An(fdsp_unop(1, y, x.release())); }
inline An operator-(An x, float y) { return An(fdsp_unop(1, -y, x.release())); }
inline An operator-(float y, An x) { return An(fdsp_unop(2, y, x.release())); }
inline An operator*(An x, float y) { return An(fdsp_unop(3, y, x.release())); }
inline An operator*(float y, An x) { return An(fdsp_unop(3, y, x.release())); }

// ---- opcodes (src/prelude.rs; F = f32)
inline An constant(std::initializer_list<float> v) { return An(fdsp_constant((int)v.size(), v.begin())); }
inline An dc(float x) { return constant({x}); }
inline An dc(float x, float y) { return constant({x, y}); }
inline An dc(float x, float y, float z) { return constant({x, y, z}); }
inline An zero() { return dc(0.0f); }
inline An pass() { return An(fdsp_pass()); }
inline An multipass(int n) { return An(fdsp_multipass(n)); }
inline An sink() { return An(fdsp_sink(1)); }
inline An multisink(int n) { return An(fdsp_sink(n)); }
inline An split(int n) { return An(fdsp_split(n)); }
inline An multisplit(int m, int n) { return An(fdsp_multisplit(m, n)); }
inline An join(int n) { return An(fdsp_join(n)); }
inline An multijoin(int m, int n) { return An(fdsp_multijoin(m, n)); }
inline An reverse(int n) { return An(fdsp_reverse(n)); }
inline An sine() { return An(fdsp_sine()); }
inline An sine_hz(float f) { return dc(f) >> sine(); }
inline An saw() { return An(fdsp_wavesynth(0, 1)); }
inline An square() { return An(fdsp_wavesynth(1, 1)); }
inline An triangle() { return An(fdsp_wavesynth(2, 1)); }
inline An organ() { return An(fdsp_wavesynth(3, 1)); }
inline An soft_saw() { return An(fdsp_wavesynth(4, 1)); }
inline An hammond() { return An(fdsp_wavesynth(5, 1)); }
inline An saw_hz(float f) { return dc(f) >> saw(); }
inline An square_hz(float f) { return dc(f) >> square(); }
inline An triangle_hz(float f) { return dc(f) >> triangle(); }
inline An noise() { return An(fdsp_noise()); }
inline An white() { return An(fdsp_noise()); }
inline An lowpass() { return An(fdsp_svf(0, 440.0f, 1.0f, 1.0f)); }
inline An lowpass_hz(float f, float q) { return An(fdsp_fixed_svf(0, f, q, 1.0f)); }
inline An highpass_hz(float f, float q) { return An(fdsp_fixed_svf(1, f, q, 1.0f)); }
inline An bandpass_hz(float f, float q) { return An(fdsp_fixed_svf(2, f, q, 1.0f)); }
inline An notch_hz(float f, float q) { return An(fdsp_fixed_svf(3, f, q, 1.0f)); }
inline An peak_hz(float f, float q) { return An(fdsp_fixed_svf(4, f, q, 1.0f)); }
inline An allpass_hz(float f, float q) { return An(fdsp_fixed_svf(5, f, q, 1.0f)); }
inline An bell_hz(float f, float q, float gain) { return An(fdsp_fixed_svf(6, f, q, gain)); }
inline An lowshelf_hz(float f, float q, float gain) { return An(fdsp_fixed_svf(7, f, q, gain)); }
inline An highshelf_hz(float f, float q, float gain) { return An(fdsp_fixed_svf(8, f, q, gain)); }
inline An biquad(float a1, float a2, float b0, float b1, float b2) { return An(fdsp_biquad(a1, a2, b0, b1, b2)); }
inline An biquad_bank() { return An(fdsp_biquad_bank()); }
inline An butterpass_hz(float f) { return An(fdsp_butterpass(f, 1)); }
inline An resonator_hz(float center, float q) { return An(fdsp_resonator(center, q, 1)); }
inline An moog() { return An(fdsp_moog(1000.0f, 0.1f, 3)); }
inline An moog_hz(float f, float q) { return An(fdsp_moog(f, q, 1)); }
inline An moog_q(float q) { return (multipass(2) | dc(q)) >> An(fdsp_moog(1000.0f, q, 3)); }
inline An fir(std::initializer_list<float> w) { return An(fdsp_fir((int)w.size(), w.begin())); }
inline An fir3(float gain) { float alpha = (gain + 1.0f) / 2.0f, beta = (1.0f - alpha) / 2.0f; return fir({beta, alpha, beta}); }
inline An tick() { return An(fdsp_tick(1)); }
inline An delay(double t) { return An(fdsp_delay(t)); }
inline An ramp() { return An(fdsp_phase_osc(0)); }
inline An ramp_hz(float f) { return dc(f) >> ramp(); }
inline An poly_saw() { return An(fdsp_phase_osc(1)); }
inline An poly_saw_hz(float f) { return dc(f) >> poly_saw(); }
inline An poly_square() { return An(fdsp_phase_osc(2)); }
inline An poly_square_hz(float f) { return dc(f) >> poly_square(); }
inline An poly_pulse() { return An(fdsp_phase_osc(3)); }
inline An poly_pulse_hz(float f, float width) { return dc(f, width) >> poly_pulse(); }
inline An reverb3_stereo(double time, double diffusion, An filter) { return An(fdsp_reverb3(time, diffusion, filter.release())); }
inline An feedback_unit(double delay, An x) { return An(fdsp_feedback_unit(delay, x.release())); }
inline An convolve(const std::vector<float>& response) { return An(fdsp_convolve(response.data(), (int)response.size())); }
inline An lowpole() { return An(fdsp_onepole(0, 440.0f, 2)); }
inline An lowpole_hz(float cutoff) { return An(fdsp_onepole(0, cutoff, 1)); }
inline An highpole() { return An(fdsp_onepole(1, 440.0f, 2)); }
inline An highpole_hz(float cutoff) { return An(fdsp_onepole(1, cutoff, 1)); }
inline An allpole() { return An(fdsp_onepole(2, 1.0f, 2)); }
inline An allpole_delay(float delay) { return An(fdsp_onepole(2, delay, 1)); }
inline An dcblock_hz(float cutoff) { return An(fdsp_onepole(3, cutoff, 1)); }
inline An dcblock() { return dcblock_hz(10.0f); }
inline An pinkpass() { return An(fdsp_onepole(4, 0.0f, 1)); }
inline An pink() { return white() >> pinkpass(); }
inline An brown() { return white() >> lowpole_hz(10.0f) * dc(13.7f); }
inline An clip() { return An(fdsp_shaper(0, 1.0f, 0.0f)); }
inline An clip_to(float lo, float hi) { return An(fdsp_shaper(1, lo, hi)); }
struct Clip { float h; }; struct ClipTo { float lo, hi; }; struct Tanh { float h; }; struct Softsign { float h; }; struct Crush { float levels; }; struct SoftCrush { float levels; };
struct Atan { float h; };
/* Adaptive::new(timescale, inner) (src/shape.rs:156-200): inner is one of the structs above (not another Adaptive) */
template <class S> struct Adaptive { double timescale; S inner; };
inline An shape(Clip s) { return An(fdsp_shaper(0, s.h, 0.0f)); }
inline An shape(ClipTo s) { return An(fdsp_shaper(1, s.lo, s.hi)); }
inline An shape(Tanh s) { return An(fdsp_shaper(2, s.h, 0.0f)); }
inline An shape(Softsign s) { return An(fdsp_shaper(3, s.h, 0.0f)); }
inline An shape(Crush s) { return An(fdsp_shaper(4, s.levels, 0.0f)); }
inline An shape(SoftCrush s) { return An(fdsp_shaper(5, s.levels, 0.0f)); }
inline An shape(Atan s) { return An(fdsp_shaper(6, s.h, 0.0f)); }
inline An follow(float response_time) { return An(fdsp_follow(0, response_time, response_time)); }
inline An afollow(float attack, float release) { return An(fdsp_follow(1, attack, release)); }
inline An morph() { return An(fdsp_morph(440.0f, 1.0f)); }
inline An morph_hz(float f, float q, float m) { return (pass() | dc(f, q, m)) >> An(fdsp_morph(f, q)); }
inline An lowrez() { return An(fdsp_rez(0.0f, 440.0f, 1.0f, 3)); }
inline An lowrez_hz(float cutoff, float q) { return An(fdsp_rez(0.0f, cutoff, q, 1)); }
inline An bandrez() { return An(fdsp_rez(1.0f, 440.0f, 1.0f, 3)); }
inline An bandrez_hz(float center, float q) { return An(fdsp_rez(1.0f, center, q, 1)); }
inline An rossler() { return An(fdsp_chaos(0)); }
inline An lorenz() { return An(fdsp_chaos(1)); }
inline An declick() { return An(fdsp_declick(0.010f)); }
inline An declick_s(float t) { return An(fdsp_declick(t)); }
/* nonlinear biquads (src/prelude.rs:2900-3110): d* = DirtyBiquad (shaped state), f* = FbBiquad (shaped feedback); the shape is any of the
   Shaper structs above. The plain forms take (audio, center, q[, gain]) at audio rate. */
struct ShapeMode { int kind; float p0, p1; double timescale; };   /* timescale > 0: Adaptive around the kind */
inline ShapeMode shape_mode(Clip s) { return {0, s.h, 0.0f}; }
inline ShapeMode shape_mode(ClipTo s) { return {1, s.lo, s.hi}; }
inline ShapeMode shape_mode(Tanh s) { return {2, s.h, 0.0f}; }
inline ShapeMode shape_mode(Softsign s) { return {3, s.h, 0.0f}; }
inline ShapeMode shape_mode(Crush s) { return {4, s.levels, 0.0f}; }
inline ShapeMode shape_mode(SoftCrush s) { return {5, s.levels, 0.0f}; }
inline ShapeMode shape_mode(Atan s) { return {6, s.h, 0.0f}; }
template <class S> inline ShapeMode shape_mode(Adaptive<S> s) {   /* a nested Adaptive lowers to kind -1, which the C ABI refuses */
    ShapeMode m = shape_mode(s.inner);
    return {m.timescale > 0.0 ? -1 : m.kind, m.p0, m.p1, s.timescale};
}
template <class S> inline An shape(Adaptive<S> s) { ShapeMode m = shape_mode(s); return An(fdsp_shaper_adaptive(m.timescale, m.kind, m.p0, m.p1)); }
inline An nl_biquad(int fb, int mode, ShapeMode m, int inputs, float center = 440.0f, float q = 1.0f, float gain = 1.0f) {
    if (m.timescale > 0.0) return An(fdsp_nl_biquad_adaptive(fb, mode, m.timescale, m.kind, m.p0, m.p1, inputs, center, q, gain));
    return An(fdsp_nl_biquad(fb, mode, m.kind, m.p0, m.p1, inputs, center, q, gain));
}
#define FDSP_NLB(NAME, FB, MODE, NIN)                                                                                   \
    template <class S> inline An NAME(S s) { return nl_biquad(FB, MODE, shape_mode(s), NIN); }
FDSP_NLB(dresonator, 0, 0, 3) FDSP_NLB(dlowpass, 0, 1, 3) FDSP_NLB(dhighpass, 0, 2, 3) FDSP_NLB(dbell, 0, 3, 4)
FDSP_NLB(fresonator, 1, 0, 3) FDSP_NLB(flowpass, 1, 1, 3) FDSP_NLB(fhighpass, 1, 2, 3) FDSP_NLB(fbell, 1, 3, 4)
#undef FDSP_NLB
template <class S> inline An dresonator_hz(S s, float c, float q) { return nl_biquad(0, 0, shape_mode(s), 1, c, q); }
template <class S> inline An dlowpass_hz(S s, float c, float q) { return nl_biquad(0, 1, shape_mode(s), 1, c, q); }
template <class S> inline An dhighpass_hz(S s, float c, float q) { return nl_biquad(0, 2, shape_mode(s), 1, c, q); }
template <class S> inline An dbell_hz(S s, float c, float q, float g) { return nl_biquad(0, 3, shape_mode(s), 1, c, q, g); }
template <class S> inline An fresonator_hz(S s, float c, float q) { return nl_biquad(1, 0, shape_mode(s), 1, c, q); }
template <class S> inline An flowpass_hz(S s, float c, float q) { return nl_biquad(1, 1, shape_mode(s), 1, c, q); }
template <class S> inline An fhighpass_hz(S s, float c, float q) { return nl_biquad(1, 2, shape_mode(s), 1, c, q); }
template <class S> inline An fbell_hz(S s, float c, float q, float g) { return nl_biquad(1, 3, shape_mode(s), 1, c, q, g); }
inline An var(float value) { return An(fdsp_var(value)); }
inline An dsf_saw() { return An(fdsp_dsf(2, 1.0f, 0.5f)); }
inline An dsf_saw_r(float roughness) { return An(fdsp_dsf(1, 1.0f, roughness)); }
inline An dsf_square() { return An(fdsp_dsf(2, 2.0f, 0.5f)); }
inline An dsf_square_r(float roughness) { return An(fdsp_dsf(1, 2.0f, roughness)); }
inline An mls_bits(int n) { return An(fdsp_mls(n)); }
inline An mls() { return mls_bits(29); }
inline An impulse(int n = 1) { return An(fdsp_impulse(n)); }
inline An tap(float min_delay, float max_delay) { return An(fdsp_tap(1, 0, min_delay, max_delay)); }
inline An multitap(int n, float min_delay, float max_delay) { return An(fdsp_tap(n, 0, min_delay, max_delay)); }
inline An tap_linear(float min_delay, float max_delay) { return An(fdsp_tap(1, 1, min_delay, max_delay)); }
inline An multitap_linear(int n, float min_delay, float max_delay) { return An(fdsp_tap(n, 1, min_delay, max_delay)); }
inline An butterpass() { return An(fdsp_butterpass(440.0f, 2)); }
inline An resonator() { return An(fdsp_resonator(440.0f, 1.0f, 3)); }
inline An feedback2(An x, An y) { return An(fdsp_feedback2(x.release(), y.release(), 0)); }
inline An fdn2(An x, An y) { return An(fdsp_feedback2(x.release(), y.release(), 1)); }
inline An pan(float p) { return An(fdsp_pan(p)); }
inline An panner() { return An(fdsp_panner()); }
inline An adsr_live(float a, float d, float s, float r) { return An(fdsp_adsr_live(a, d, s, r)); }
// closures of the signal, run per sample on the device (DESIGN.md §2 / row f.12): the closure as text, captured values by name, e.g.
//   map("|x| tanh(x[0] * drive)", 1, 1, {{"drive", 0.7f}})
// A refused text throws Error with the token and its column (FDSP_ERR_ARITY for arity mismatches, else FDSP_ERR_ARG).
using Captures = std::initializer_list<std::pair<const char*, float>>;
namespace detail {
inline An closure_node(fdsp_node* h) {
  if (h) return An(h);
  const std::string e = fdsp_last_error();
  throw Error(e.find(": arity mismatch") != std::string::npos ? FDSP_ERR_ARITY : FDSP_ERR_ARG, e);
}
struct CaptureArrays {
  std::vector<const char*> names; std::vector<float> values;
  explicit CaptureArrays(Captures c) { for (const auto& p : c) { names.push_back(p.first); values.push_back(p.second); } }
};
}  // namespace detail
inline An map(const char* closure, int inputs, int outputs, Captures captures = {}) {
  detail::CaptureArrays c(captures);
  return detail::closure_node(fdsp_map(inputs, outputs, closure, (int)c.names.size(), c.names.data(), c.values.data()));
}
inline An shape_fn(const char* closure, Captures captures = {}) {
  detail::CaptureArrays c(captures);
  return detail::closure_node(fdsp_shape_fn(closure, (int)c.names.size(), c.names.data(), c.values.data()));
}
inline An envelope_in(const char* closure, int inputs, int outputs = 1, Captures captures = {}) {
  detail::CaptureArrays c(captures);
  return detail::closure_node(fdsp_envelope_in(0.002, inputs, outputs, closure, (int)c.names.size(), c.names.data(), c.values.data()));
}
inline An lfo_in(const char* closure, int inputs, int outputs = 1, Captures captures = {}) { return envelope_in(closure, inputs, outputs, captures); }
inline An envelope2(const char* closure, int outputs = 1, Captures captures = {}) { return envelope_in(closure, 1, outputs, captures); }
inline An lfo2(const char* closure, int outputs = 1, Captures captures = {}) { return envelope_in(closure, 1, outputs, captures); }
inline An envelope3(const char* closure, int outputs = 1, Captures captures = {}) { return envelope_in(closure, 2, outputs, captures); }
inline An lfo3(const char* closure, int outputs = 1, Captures captures = {}) { return envelope_in(closure, 2, outputs, captures); }
inline An feedback(An x) { return An(fdsp_feedback(x.release(), 0)); }
inline An fdn(An x) { return An(fdsp_feedback(x.release(), 1)); }
template <class F> An stacki(int n, F f) { std::vector<fdsp_node*> v; for (int i = 0; i < n; i++) v.push_back(f(i).release()); return An(fdsp_multi(30, 0, n, v.data())); }
template <class F> An busi(int n, F f) { std::vector<fdsp_node*> v; for (int i = 0; i < n; i++) v.push_back(f(i).release()); return An(fdsp_multi(28, 0, n, v.data())); }
template <class F> An sumi(int n, F f) { std::vector<fdsp_node*> v; for (int i = 0; i < n; i++) v.push_back(f(i).release()); return An(fdsp_multi(31, 0, n, v.data())); }
template <class F> An branchi(int n, F f) { std::vector<fdsp_node*> v; for (int i = 0; i < n; i++) v.push_back(f(i).release()); return An(fdsp_multi(33, 0, n, v.data())); }
template <class F> An pipei(int n, F f) { std::vector<fdsp_node*> v; for (int i = 0; i < n; i++) v.push_back(f(i).release()); return An(fdsp_multi(32, 0, n, v.data())); }
template <class F> An sumf(int n, F f) { std::vector<fdsp_node*> v; for (int i = 0; i < n; i++) v.push_back(f(n > 1 ? (float)((double)i / (double)(n - 1)) : 0.5f).release()); return An(fdsp_multi(31, 0, n, v.data())); }
inline An pulse() { return An(fdsp_pulse()); }                                         // inputs (frequency, width)
inline An phase_synth(int table) { return An(fdsp_phase_synth(table)); }               // An(PhaseSynth::new(table))
inline An rotate(float angle, float gain) { return An(fdsp_rotate(angle, gain)); }
inline An mixer(int inputs, int outputs, std::initializer_list<float> matrix) { return (int)matrix.size() == inputs * outputs ? An(fdsp_mixer(inputs, outputs, matrix.begin())) : An(nullptr); }
struct Meter { int kind; double timescale; static Meter Sample() { return {0, 0.0}; } static Meter Peak(double t) { return {1, t}; } static Meter Rms(double t) { return {2, t}; } };
inline An meter(Meter m) { return An(fdsp_meter(m.kind, m.timescale)); }
// playwave(&wave, channel, loop): `samples` = wave.channel(channel); loop_point < 0 = None
inline An playwave(const std::vector<float>& samples, long long loop_point = -1) { return An(fdsp_playwave(samples.data(), samples.size(), 0, samples.size(), loop_point)); }
inline An playwave_at(const std::vector<float>& samples, size_t start, size_t end, long long loop_point = -1) { return An(fdsp_playwave(samples.data(), samples.size(), start, end, loop_point)); }
inline An limiter(float attack_time, float release_time) { return An(fdsp_limiter(1, attack_time, release_time)); }
inline An limiter_stereo(float attack_time, float release_time) { return An(fdsp_limiter(2, attack_time, release_time)); }
// envelope(|t| ...) / lfo(|t| ...) (src/prelude.rs:580-612): a capture-less lambda or function `void f(double t, double* out, void* user)`;
// the closure runs on the host when the graph is lowered, at the reference's sample points, up to `horizon` seconds
inline An envelope(fdsp_envelope_fn f, int outputs = 1, void* user = nullptr, double horizon = 10.0, bool time64 = false) { return An(fdsp_envelope(0.002, outputs, time64 ? 1 : 0, f, user, horizon)); }
inline An lfo(fdsp_envelope_fn f, int outputs = 1, void* user = nullptr, double horizon = 10.0, bool time64 = false) { return envelope(f, outputs, user, horizon, time64); }
// flanger / phaser (src/prelude.rs:2719-2753): the delay (phase) closure is a closure of time and lowers like `lfo`. phaser's closure
// returns the allpole delay itself here: lerp(2, 20, clamp01(phase_f(t))) of the reference is the caller's to apply.
inline An flanger(float feedback_amount, float minimum_delay, float maximum_delay, fdsp_envelope_fn delay_f, void* user = nullptr, double horizon = 10.0) {
  return pass() & feedback2((pass() | lfo(delay_f, 1, user, horizon)) >> tap(minimum_delay, maximum_delay), shape(Tanh{feedback_amount}));
}
enum class Fade { Power = 0, Smooth = 1 };                                                 // src/sequencer.rs:35-52
inline An slot(An unit) { return An(fdsp_slot(unit.release())); }                             // Slot::new: replaceable with a crossfade (Bank::slot_set)
// one Sequencer event as a voice (Sequencer::push, src/sequencer.rs:319-345): a Bank of events is the sequencer
inline An event(An unit, double start_time, double end_time, Fade ease = Fade::Smooth, double fade_in = 0.0, double fade_out = 0.0) {
  return An(fdsp_event(unit.release(), start_time, end_time, (int)ease, fade_in, fade_out));
}
// an event of a `Sequencer::new(0, outputs, ReplayMode::Loop(loop_seconds))` (src/sequencer.rs:219-229)
inline An event_loop(An unit, double start_time, double end_time, double loop_seconds, Fade ease = Fade::Smooth, double fade_in = 0.0, double fade_out = 0.0) {
  return An(fdsp_event_loop(unit.release(), start_time, end_time, (int)ease, fade_in, fade_out, loop_seconds));
}
inline An oversample(An x) { return An(fdsp_oversample(x.release())); }                // x at twice the sample rate
inline An resample(An x) { return An(fdsp_resample(x.release())); }                    // input = speed

// ---- src/math.rs helpers used by the reverbs, in the reference's precision
inline float lerp(float a, float b, float t) { return a * (1.0f - t) + b * t; }
inline float smooth9(float x) { float x2 = x * x; return ((((70.0f * x - 315.0f) * x + 540.0f) * x - 420.0f) * x + 126.0f) * x2 * x2 * x; }
inline double db_amp(double db) { return std::exp((db / 20.0) * std::log(10.0)); }
// src/prelude.rs:1732-1762 and :1873-1946: the FDN reverbs as the reference composes them
inline An reverb_stereo(double room_size, double time, float damping) {
  static const double delays[32] = {0.073904, 0.052918, 0.066238, 0.066387, 0.037783, 0.080073, 0.050961, 0.075900, 0.043646, 0.072095, 0.056194,
                                    0.045961, 0.058934, 0.068016, 0.047529, 0.058156, 0.072972, 0.036084, 0.062715, 0.076377, 0.044339, 0.076725,
                                    0.077884, 0.046126, 0.067741, 0.049800, 0.051709, 0.082923, 0.070121, 0.079315, 0.055039, 0.081859};
  const float a = (float)std::pow(db_amp(-60.0), 0.03 * room_size / 10.0 / time);
  const float gain = 1.0f - damping, alpha = (gain + 1.0f) / 2.0f, beta = (1.0f - alpha) / 2.0f;
  An line = stacki(32, [&](int i) { return delay(delays[i] * room_size / 10.0) >> fir({beta * a, alpha * a, beta * a}); });
  return multisplit(2, 16) >> fdn(std::move(line)) >> sumf(32, [](float x) { return pan(lerp(-1.0f, 1.0f, smooth9(x))); }) * dc(1.0f / 16.0f, 1.0f / 16.0f);
}
inline An reverb4_stereo_delays(const float (&delays)[32], double time) {
  const float a = (float)std::pow(db_amp(-60.0), 0.03 * 10.0 / 10.0 / time);
  An line1 = stacki(16, [&](int i) { return delay((double)delays[i]) >> fir({-a / 4.0f, -a / 2.0f, -a / 4.0f}); });
  An line2 = stacki(16, [&](int i) { return delay((double)delays[16 + i]) >> fir({-a / 4.0f, -a / 2.0f, -a / 4.0f}); });
  return multisplit(2, 8) >> fdn(std::move(line1)) >> multijoin(2, 8) >> multisplit(2, 8) >> fdn(std::move(line2))
         >> sumf(16, [](float x) { return pan(lerp(-1.0f, 1.0f, smooth9(x))); }) * dc(1.0f / 4.0f, 1.0f / 4.0f);
}
inline An reverb4_stereo(double room_size, double time) {
  float d[32] = {0.059326634f, 0.04778291f, 0.06995449f, 0.0393001f, 0.041604012f, 0.06215825f, 0.052269846f, 0.043227978f, 0.06966107f, 0.031615064f, 0.068442f,
                 0.037332155f, 0.032944717f, 0.034493037f, 0.06787566f, 0.038824916f, 0.068260126f, 0.068044715f, 0.0688076f, 0.066724524f, 0.051293883f, 0.06023173f,
                 0.040897705f, 0.031507637f, 0.060309593f, 0.049584292f, 0.04532072f, 0.056379095f, 0.035180368f, 0.041291796f, 0.046129026f, 0.05504605f};
  const float k = std::fmax((float)room_size, 15.0f) / 10.0f;
  for (float& x : d) x *= k;
  return reverb4_stereo_delays(d, time);
}

// ---- the voice bank as an AudioUnit
class Bank {
  fdsp_bank* b_ = nullptr;

 public:
  // consumes the voices; `mix`: sum the voices (outputs() == channels), else per-voice rows (outputs() == V * channels)
  Bank(std::vector<An>& voices, int device = 0, bool per_voice = false, bool mix = true) {
    std::vector<fdsp_node*> hs;
    for (auto& v : voices) hs.push_back(v.release());
    voices.clear();
    check(fdsp_bank_create(hs.data(), (uint32_t)hs.size(), device, (per_voice ? FDSP_OUT_VOICES : 0) | (mix ? FDSP_OUT_MIX : 0), &b_));
  }
  Bank(const Bank&) = delete;
  Bank& operator=(const Bank&) = delete;
  ~Bank() { fdsp_bank_destroy(b_); }
  int inputs() const { return fdsp_bank_inputs(b_); }
  int outputs() const { return fdsp_bank_outputs(b_); }
  uint32_t voices() const { return fdsp_bank_voices(b_); }
  void set_sample_rate(double sr) { check(fdsp_bank_set_sample_rate(b_, sr)); }
  void reset() { check(fdsp_bank_reset(b_)); }
  // AudioUnit::set on one voice: `kind` is the Parameter index of src/setting.rs (fundsp_b200.h), `address` = {type, value} pairs
  // (type 1 Index, 2 Node) exactly as in fdsp_node_set; e.g. set(7, FDSP_P_CENTER_Q, {2500.f, 3.f}, {{1, 0}, {1, 1}})
  void set(uint32_t voice, int kind, std::initializer_list<float> values, std::initializer_list<std::pair<int, int64_t>> address = {}, uint64_t seed = 0) {
    std::vector<int64_t> a;
    for (auto& p : address) { a.push_back(p.first); a.push_back(p.second); }
    check(fdsp_bank_set(b_, voice, kind, values.begin(), (int)values.size(), seed, a.empty() ? nullptr : a.data(), (int)address.size()));
  }
  void allocate(uint64_t max_samples = 64) { check(fdsp_bank_allocate(b_, max_samples)); }
  // sequencer banks: Sequencer::time / edit / push on a running bank (a pushed event reuses the slot of a finished event of its class)
  double time() const { return fdsp_bank_time(b_); }
  void edit_event(uint32_t voice, double end_time, double fade_out) { check(fdsp_bank_edit_event(b_, voice, end_time, fade_out)); }
  uint32_t push_event(An ev) { uint32_t v = 0; check(fdsp_bank_push_event(b_, ev.release(), &v)); return v; }
  void replace_voice(uint32_t voice, An unit) { check(fdsp_bank_replace_voice(b_, voice, unit.release())); }
  void slot_set(uint32_t voice, Fade fade, double fade_time, An unit) { check(fdsp_bank_slot_set(b_, voice, (int)fade, fade_time, unit.release())); }   // Slot::set
  uint32_t add_voice(An unit) { uint32_t v = 0; check(fdsp_bank_add_voice(b_, unit.release(), &v)); return v; }   // grows the bank; the others keep their state
  // AudioUnit::process: buffers are [channel][64]
  void process(uint32_t size, const float* input, float* output) { check(fdsp_bank_process(b_, size, input, output)); }
  // Wave::render / Wave::filter: buffers are [channel][n]
  void render(uint64_t n, const float* input, float* out_voices, float* out_mix) { check(fdsp_bank_render(b_, n, input, out_voices, out_mix)); }
  fdsp_bank* get() { return b_; }
};

// fundsp::prelude64: the opcodes whose prelude64 type keeps f64 state (Sine<f64>, the SVFs, biquads and one-poles). Everything else is the
// f32 opcode above; `using namespace fundsp_b200::prelude64;` after `using namespace fundsp_b200;` selects these where the names meet.
namespace prelude64 {
inline An sine() { return An(fdsp_sine_f64()); }
inline An sine_hz(float f) { return dc(f) >> sine(); }
namespace detail {
inline An svf(int mode) { return An(fdsp_svf_f64(mode, 440.0f, 1.0f, 1.0f)); }
inline An svf_hz(int mode, float f, float q, float gain = 1.0f) { return An(fdsp_fixed_svf_f64(mode, f, q, gain)); }
inline An svf_q(int mode, float q) { return (multipass(2) | dc(q)) >> An(fdsp_svf_f64(mode, 440.0f, q, 1.0f)); }
inline An svf_q(int mode, float q, float gain) { return (multipass(2) | dc(q, gain)) >> An(fdsp_svf_f64(mode, 440.0f, q, gain)); }
}  // namespace detail
inline An lowpass() { return detail::svf(0); }
inline An lowpass_hz(float f, float q) { return detail::svf_hz(0, f, q); }
inline An lowpass_q(float q) { return detail::svf_q(0, q); }
inline An highpass() { return detail::svf(1); }
inline An highpass_hz(float f, float q) { return detail::svf_hz(1, f, q); }
inline An highpass_q(float q) { return detail::svf_q(1, q); }
inline An bandpass() { return detail::svf(2); }
inline An bandpass_hz(float f, float q) { return detail::svf_hz(2, f, q); }
inline An bandpass_q(float q) { return detail::svf_q(2, q); }
inline An notch() { return detail::svf(3); }
inline An notch_hz(float f, float q) { return detail::svf_hz(3, f, q); }
inline An notch_q(float q) { return detail::svf_q(3, q); }
inline An peak() { return detail::svf(4); }
inline An peak_hz(float f, float q) { return detail::svf_hz(4, f, q); }
inline An peak_q(float q) { return detail::svf_q(4, q); }
inline An allpass() { return detail::svf(5); }
inline An allpass_hz(float f, float q) { return detail::svf_hz(5, f, q); }
inline An allpass_q(float q) { return detail::svf_q(5, q); }
inline An bell() { return detail::svf(6); }
inline An bell_hz(float f, float q, float gain) { return detail::svf_hz(6, f, q, gain); }
inline An bell_q(float q, float gain) { return detail::svf_q(6, q, gain); }
inline An lowshelf() { return detail::svf(7); }
inline An lowshelf_hz(float f, float q, float gain) { return detail::svf_hz(7, f, q, gain); }
inline An lowshelf_q(float q, float gain) { return detail::svf_q(7, q, gain); }
inline An highshelf() { return detail::svf(8); }
inline An highshelf_hz(float f, float q, float gain) { return detail::svf_hz(8, f, q, gain); }
inline An highshelf_q(float q, float gain) { return detail::svf_q(8, q, gain); }
inline An biquad(float a1, float a2, float b0, float b1, float b2) { return An(fdsp_biquad_f64(a1, a2, b0, b1, b2)); }
inline An butterpass() { return An(fdsp_butterpass_f64(440.0f, 2)); }
inline An butterpass_hz(float f) { return An(fdsp_butterpass_f64(f, 1)); }
inline An resonator() { return An(fdsp_resonator_f64(440.0f, 1.0f, 3)); }
inline An resonator_hz(float center, float q) { return An(fdsp_resonator_f64(center, q, 1)); }
inline An lowpole() { return An(fdsp_onepole_f64(0, 440.0f, 2)); }
inline An lowpole_hz(float cutoff) { return An(fdsp_onepole_f64(0, cutoff, 1)); }
inline An highpole() { return An(fdsp_onepole_f64(1, 440.0f, 2)); }
inline An highpole_hz(float cutoff) { return An(fdsp_onepole_f64(1, cutoff, 1)); }
inline An allpole() { return An(fdsp_onepole_f64(2, 1.0f, 2)); }
inline An allpole_delay(float delay) { return An(fdsp_onepole_f64(2, delay, 1)); }
inline An dcblock_hz(float cutoff) { return An(fdsp_onepole_f64(3, cutoff, 1)); }
inline An dcblock() { return dcblock_hz(10.0f); }
inline An pinkpass() { return An(fdsp_onepole_f64(4, 0.0f, 1)); }
inline An pink() { return noise() >> pinkpass(); }
inline An brown() { return noise() >> lowpole_hz(10.0f) * dc(13.7f); }
}  // namespace prelude64

}  // namespace fundsp_b200

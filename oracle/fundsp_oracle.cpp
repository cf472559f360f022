// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h). C ABI over the CPU restatement in fo_nodes.h so
// that tests/ (ctypes) and bench.py's cpu_baseline leg can drive it. Handles are heap `fo::Node*`;
// combinators CONSUME their children (like Rust move semantics); use fo_clone to reuse a node.
//
// Prelude composites restated here (paths relative to the reference crate (SamiPerttu/fundsp v0.23.0)):
//   sine_hz  src/prelude.rs:349-351      saw_hz etc. src/prelude.rs:2051-2089
//   fir3     src/prelude.rs:863-867      reverb_stereo src/prelude.rs:1732-1762
//   moog_q   src/prelude.rs:559-561      Wave::render src/wave.rs:441-466, Wave::filter :518-565
#include "fo_nodes.h"
#include "fo_shapes.h"   // atanf_ and wide_atanf, for fo_libm_eval
#include <thread>

using namespace fo;

#define API extern "C" __attribute__((visibility("default")))

API const char* fo_about() { return "fundsp oracle: CPU restatement of SamiPerttu/fundsp v0.23.0 block path (test infrastructure)"; }

// ---- math helpers exported for golden-vector tests
API double fo_rnd1(uint64_t x) { return rnd1(x); }
API uint64_t fo_hash1(uint64_t x) { return hash1(x); }
API uint64_t fo_attohash(uint64_t state, uint64_t data) { return AttoHash(state).hash(data).state; }
API uint32_t fo_hash32x(uint32_t x) { return hash32x(x); }
API float fo_wide_sinf(float x) { return wide_sinf(x); }
API float fo_wide_floorf(float x) { return wide_floorf(x); }
API float fo_lerpf(float a, float b, float t) { return lerpf(a, b, t); }
API double fo_lerpd(double a, double b, double t) { return lerpd(a, b, t); }
API double fo_delerpd(double a, double b, double x) { return delerpd(a, b, x); }
API float fo_xerpf(float a, float b, float t) { return xerpf(a, b, t); }
API double fo_xerpd(double a, double b, double t) { return xerpd(a, b, t); }
API double fo_db_amp(double db) { return db_ampd(db); }
API float fo_smooth9f(float x) { return smooth9f(x); }
API void fo_set_denormal_emulation(int on) { denormal_emulation_enabled() = on != 0; if (!on) _mm_setcsr(0x1f80); }
API void fo_restore_denormals() { _mm_setcsr(0x1f80); }

// ---- wavetable introspection: kind 0..5; returns number of tables; per-table pitch/len/data
API int fo_wavetable_count(int kind) { return (int)global_table(kind).table.size(); }
API float fo_wavetable_pitch(int kind, int i) { return global_table(kind).table[i].first; }
API int fo_wavetable_len(int kind, int i) { return (int)global_table(kind).table[i].second.size(); }
API const float* fo_wavetable_data(int kind, int i) { return global_table(kind).table[i].second.data(); }
// test-only: read kind `kind` from the given tables (n tables, pitch[i], len[i] floats each, concatenated in `data`) instead of this
// file's own builder, until fo_wavetable_restore(kind). Call neither while a node renders (fo_nodes.h installed_table).
API int fo_wavetable_install(int kind, int n, const float* pitch, const int* len, const float* data) {
  if (kind < 0 || kind > 5 || n < 3) return -1;
  std::unique_ptr<Wavetable> w(new Wavetable());
  for (int i = 0; i < n; i++) {
    if (len[i] < 2 || (len[i] & (len[i] - 1))) return -1;   // the read masks indices: power-of-two lengths only
    w->table.emplace_back(pitch[i], std::vector<float>(data, data + len[i]));
    data += len[i];
  }
  installed_table(kind) = std::move(w);
  return 0;
}
API void fo_wavetable_restore(int kind) { if (kind >= 0 && kind <= 5) installed_table(kind).reset(); }

// ---- leaves
API Node* fo_constant(int n, const float* v) { return new Constant(std::vector<float>(v, v + n)); }
API Node* fo_pass() { return new MultiPass(1, true); }
API Node* fo_multipass(int n) { return new MultiPass(n, false); }
API Node* fo_sink(int n) { return new Sink(n); }
API Node* fo_split(int n) { return new MultiSplit(1, n, true); }
API Node* fo_multisplit(int m, int n) { return new MultiSplit(m, n, false); }
API Node* fo_join(int n) { return new MultiJoin(1, n, true); }
API Node* fo_multijoin(int m, int n) { return new MultiJoin(m, n, false); }
API Node* fo_reverse(int n) { return new Reverse(n); }
API Node* fo_sine() { return new Sine(); }
API Node* fo_wavesynth(int kind, int outputs) { return new WaveSynth(kind, outputs); }
API Node* fo_noise() { return new Noise(); }
API Node* fo_fixed_svf(int mode, float cutoff, float q, float gain) { return new Svf(mode, true, cutoff, q, gain); }
API Node* fo_svf(int mode, float cutoff, float q, float gain) { return new Svf(mode, false, cutoff, q, gain); }
API Node* fo_biquad(float a1, float a2, float b0, float b1, float b2) { BiquadCoefs c; c.a1 = a1; c.a2 = a2; c.b0 = b0; c.b1 = b1; c.b2 = b2; return new Biquad(c); }
API Node* fo_biquad_bank() { return new BiquadBank(); }
API Node* fo_butterpass(float cutoff, int nin) { return new ButterLowpass(cutoff, nin); }
API Node* fo_resonator(float center, float q, int nin) { return new Resonator(center, q, nin); }
API Node* fo_moog(float cutoff, float q, int nin) { return new Moog(cutoff, q, nin); }
API Node* fo_fir(int n, const float* w) { return new Fir(std::vector<float>(w, w + n)); }
API Node* fo_tick_node(int n) { return new TickNode(n); }
API Node* fo_delay(double t) { return new Delay(t); }
API Node* fo_allnest(float coefficient, Node* x, int nin) { return new AllNest(coefficient, x, nin); }
API Node* fo_pan(float value) { return new Panner(value, 1); }
API Node* fo_panner() { return new Panner(0.0f, 2); }
API Node* fo_adsr_live(float a, float d, float s, float r) { return new AdsrLive(a, d, s, r); }
API Node* fo_phase_osc(int kind) { return new PhaseOsc(kind); }   // 0 ramp, 1 poly_saw, 2 poly_square, 3 poly_pulse
// restated libm entry points, for the accuracy and sweep tests
// (fn: 0 sinf 1 cosf 2 tanf 3 tanhf 4 expm1f 5 expf 6 powf(x, y) 7 atanf 8 wide_sinf 9 wide_atanf)
API void fo_libm_eval(int fn, const float* x, const float* y, float* out, int64_t n) {
  for (int64_t i = 0; i < n; i++) {
    switch (fn) {
      case 0: out[i] = m::sinf_(x[i]); break;
      case 1: out[i] = m::cosf_(x[i]); break;
      case 2: out[i] = m::tanf_(x[i]); break;
      case 3: out[i] = m::tanhf_(x[i]); break;
      case 4: out[i] = m::expm1f_(x[i]); break;
      case 5: out[i] = m::expf_(x[i]); break;
      case 7: out[i] = m::atanf_(x[i]); break;
      case 8: out[i] = wide_sinf(x[i]); break;
      case 9: out[i] = wide_atanf(x[i]); break;
      default: out[i] = m::powf_(x[i], y[i]); break;
    }
  }
}
API Node* fo_reverb3(double time, double diffusion, Node* filter) { return new Reverb85(time, diffusion, filter); }   // reverb3_stereo (src/prelude.rs:1858-1864)
API Node* fo_feedback_unit(double delay, Node* x) { return new FeedbackUnit(delay, x); }
API Node* fo_convolve(const float* response, int n) { return new Convolver(std::vector<float>(response, response + (n > 0 ? n : 0))); }
API Node* fo_onepole(int kind, float param, int inputs) { return new OnePole(kind, param, inputs); }   // 0 lowpole 1 highpole 2 allpole 3 dcblock 4 pinkpass
API Node* fo_shaper(int kind, float p0, float p1) { return new Shaper(kind, p0, p1); }   // 0 clip 1 clip_to 2 tanh 3 softsign 4 crush 5 soft_crush
API Node* fo_follow(int asymmetric, float attack, float release) { return new Follower(asymmetric != 0, attack, asymmetric ? release : attack); }
API Node* fo_morph(float cutoff, float q) { return new Morph(cutoff, q); }
API Node* fo_rez(float bandpass, float cutoff, float q, int inputs) { return new Rez(bandpass, cutoff, q, inputs); }
API Node* fo_chaos(int kind) { return new Chaos(kind); }   // 0 rossler, 1 lorenz
API Node* fo_declick(float duration) { return new Declick(duration); }
API Node* fo_slot(Node* unit) { return new Slot(unit); }
API void fo_slot_set(Node* slot, int fade, double fade_time, Node* unit) { static_cast<Slot*>(slot)->set(fade, fade_time, unit); }
API Node* fo_oversample(Node* x) { return new Oversampler(x); }
API Node* fo_monitor() { return new MultiPass(1, true, 56); }
API Node* fo_envelope(double interval, int outputs, int time_f64, EnvelopeFn f, void* user) {
  if (time_f64) return new Envelope<double>(interval, outputs, f, user);
  return new Envelope<float>((float)interval, outputs, f, user);
}
// Sequencer (src/sequencer.rs): mode 0 ReplayMode::All, 1 None, 2 Loop(loop_time); fade_ease 0 Fade::Power, 1 Fade::Smooth
API Node* fo_sequencer(int inputs, int outputs, int mode, double loop_time) { return new Sequencer(inputs, outputs, mode, loop_time); }
API uint64_t fo_sequencer_push(Node* s, double start, double end, int ease, double fade_in, double fade_out, Node* unit) { return static_cast<Sequencer*>(s)->push(start, end, ease, fade_in, fade_out, unit); }
API uint64_t fo_sequencer_push_relative(Node* s, double start, double end, int ease, double fade_in, double fade_out, Node* unit) { return static_cast<Sequencer*>(s)->push_relative(start, end, ease, fade_in, fade_out, unit); }
API void fo_sequencer_edit(Node* s, uint64_t id, double end_time, double fade_out) { static_cast<Sequencer*>(s)->edit(id, end_time, fade_out); }
API void fo_sequencer_edit_relative(Node* s, uint64_t id, double end_time, double fade_out) { static_cast<Sequencer*>(s)->edit_relative(id, end_time, fade_out); }
API double fo_sequencer_time(Node* s) { return static_cast<Sequencer*>(s)->time; }
API Node* fo_limiter(int channels, float attack, float release) { return new Limiter(channels, attack, release); }
API Node* fo_meter(int kind, double timescale) { return new MeterNode(kind, timescale); }
API Node* fo_playwave(const float* samples, uint64_t length, uint64_t start, uint64_t end, int64_t loop_point) {
  auto w = std::make_shared<std::vector<float>>(samples, samples + length);
  return new WavePlayer(std::move(w), (size_t)start, (size_t)end, loop_point >= 0, loop_point >= 0 ? (size_t)loop_point : 0);
}
API Node* fo_resample(Node* x) { return new Resample(x); }
API Node* fo_phase_synth(int kind) { return new PhaseSynth(kind); }
API Node* fo_pulse() { return new PulseWave(); }
API Node* fo_mixer(int inputs, int outputs, const float* matrix) { return new Mixer(inputs, outputs, matrix); }
API Node* fo_rotate(float angle, float gain) {   // src/prelude.rs:2876-2884
  const float c = m::cosf_(angle), s = m::sinf_(angle);
  const float w[4] = {c * gain, -s * gain, s * gain, c * gain};
  return new Mixer(2, 2, w);
}
API Node* fo_nl_biquad(int fb, int mode, int shape_kind, float p0, float p1, int inputs, float center, float q, float gain) {
  return new NlBiquad(fb != 0, mode, shape_kind, p0, p1, inputs, center, q, gain);
}
API Node* fo_var(float value) { return new Var(value); }
API Node* fo_dsf(int inputs, float harmonic_spacing, float roughness) { return new Dsf(inputs, harmonic_spacing, roughness); }
API Node* fo_mls(int bits) { return new Mls((uint32_t)bits); }
API Node* fo_impulse(int n) { return new Impulse(n); }
API Node* fo_tap(int ntaps, int linear, float min_delay, float max_delay) { return new Tap(ntaps, linear != 0, min_delay, max_delay); }
API Node* fo_feedback2(Node* x, Node* y, int hadamard_) { return new Feedback2(x, y, hadamard_ != 0); }
// BiquadCoefs constructors (src/biquad.rs:27-116), f32: kind 0 butter_lowpass, 1 resonator, 2 lowpass, 3 highpass, 4 bell
API void fo_biquad_coefs(int kind, float sr, float f, float q, float gain, float* out5) {
  BiquadCoefs c;
  switch (kind) { case 0: c = biquad_butter_lowpass(sr, f); break; case 1: c = biquad_resonator(sr, f, q); break;
    case 2: c = biquad_lowpass(sr, f, q); break; case 3: c = biquad_highpass(sr, f, q); break; default: c = biquad_bell(sr, f, q, gain); }
  out5[0] = c.a1; out5[1] = c.a2; out5[2] = c.b0; out5[3] = c.b1; out5[4] = c.b2;
}

// ---- combinators (consume children)
API Node* fo_pipe(Node* x, Node* y) { return new Pipe(x, y); }
API Node* fo_stack(Node* x, Node* y) { return new Stack(x, y); }
API Node* fo_branch(Node* x, Node* y) { return new Branch(x, y); }
API Node* fo_bus(Node* x, Node* y) { return new Bus(x, y); }
API Node* fo_thru(Node* x) { return new Thru(x); }
API Node* fo_binop(int op, Node* x, Node* y) { return new Binop(op, x, y); }
API Node* fo_unop(int kind, float scalar, Node* x) { return new Unop(kind, scalar, x); }
API Node* fo_multi(int kind, int op, int n, Node** nodes) { return new Multi(kind, op, std::vector<Node*>(nodes, nodes + n)); }
API Node* fo_feedback(Node* x, int hadamard_) { return new Feedback(x, hadamard_ != 0); }

// ---- prelude composites
API Node* fo_sine_hz(float f) { float v = f; return new Pipe(new Constant({v}), new Sine()); }
API Node* fo_wave_hz(int kind, float f) { float v = f; return new Pipe(new Constant({v}), new WaveSynth(kind, 1)); }
API Node* fo_fir3(float gain) {
  float alpha = (gain + 1.0f) / 2.0f;
  float beta = (1.0f - alpha) / 2.0f;
  return new Fir({beta, alpha, beta});
}
API Node* fo_moog_q(float q) {
  return new Pipe(new Stack(new MultiPass(2, false), new Constant({q})), new Moog(1000.0f, q, 3));
}
API Node* fo_reverb_stereo(double room_size, double time, double damping) {
  static const double DELAYS[32] = {
      0.073904, 0.052918, 0.066238, 0.066387, 0.037783, 0.080073, 0.050961, 0.075900, 0.043646,
      0.072095, 0.056194, 0.045961, 0.058934, 0.068016, 0.047529, 0.058156, 0.072972, 0.036084,
      0.062715, 0.076377, 0.044339, 0.076725, 0.077884, 0.046126, 0.067741, 0.049800, 0.051709,
      0.082923, 0.070121, 0.079315, 0.055039, 0.081859};
  float a = (float)pow(db_ampd(-60.0), 0.03 * room_size / 10.0 / time);
  float gain = 1.0f - (float)damping;
  float alpha = (gain + 1.0f) / 2.0f;
  float beta = (1.0f - alpha) / 2.0f;
  std::vector<float> weights = {beta * a, alpha * a, beta * a};
  std::vector<Node*> lines;
  for (int i = 0; i < 32; i++) lines.push_back(new Pipe(new Delay(DELAYS[i] * room_size / 10.0), new Fir(weights)));
  Node* line = new Multi(M_STACK, 0, lines);
  Node* reverb = new Feedback(line, true);
  std::vector<Node*> pans;
  for (int i = 0; i < 32; i++) {
    float x = (float)((double)i / 31.0);
    pans.push_back(new Panner(lerpf(-1.0f, 1.0f, smooth9f(x)), 1));
  }
  Node* sum = new Multi(M_REDUCE, OP_ADD, pans);
  // `>>` binds tighter than `*` is false in Rust: `a >> b >> sumf(..) * dc(..)` parses as a >> b >> (sumf * dc)
  Node* scaled = new Binop(OP_MUL, sum, new Constant({1.0f / 16.0f, 1.0f / 16.0f}));
  return new Pipe(new Pipe(new MultiSplit(2, 16, false), reverb), scaled);
}

// ---- An<X> builder methods (src/combinator.rs:263-286)
API void fo_phase(Node* n, float phase) { Setting s; s.kind = P_PHASE; s.v[0] = phase; s.address.push_back({1, 1}); n->set(s); n->reset(); }
API void fo_seed(Node* n, uint64_t seed) { Setting s; s.kind = P_SEED; s.seed = seed; s.address.push_back({1, 0}); n->set(s); n->reset(); }
// generic Setting: addr entries are (type,value) pairs, type 1 = Index, 2 = Node
API void fo_set(Node* n, int kind, const float* v, int nv, uint64_t seed, const int64_t* addr, int naddr) {
  Setting s; s.kind = kind; s.seed = seed;
  for (int i = 0; i < nv && i < 5; i++) s.v[i] = v[i];
  for (int i = 0; i < naddr; i++) s.address.push_back({(int)addr[2 * i], (uint64_t)addr[2 * i + 1]});
  n->set(s);
}

// ---- unit interface
API int fo_inputs(Node* n) { return n->inputs(); }
API int fo_outputs(Node* n) { return n->outputs(); }
API uint64_t fo_id(Node* n) { return n->id(); }
API void fo_reset(Node* n) { n->reset(); }
API void fo_set_sample_rate(Node* n, double sr) { n->set_sample_rate(sr); }
API void fo_tick(Node* n, const float* in, float* out) { n->tick(in, out); }
API void fo_process(Node* n, int size, const float* in, float* out) { n->process(size, in, out); }
API uint64_t fo_ping(Node* n, int probe, uint64_t hash) { return n->ping(probe != 0, AttoHash(hash)).state; }
// leaf hashes in ping order, as assigned by the node's own constructor-time ping (re-pings with the probe hash)
API int fo_leaf_hashes(Node* n, uint64_t* out, int max) {
  std::vector<uint64_t> t; Node::ping_trace() = &t;
  AttoHash h = n->ping(true, AttoHash(n->id())); n->ping(false, h);
  Node::ping_trace() = nullptr;
  for (int i = 0; i < (int)t.size() && i < max; i++) out[i] = t[i];
  return (int)t.size();
}
API void fo_set_hash(Node* n, uint64_t h) { n->set_hash(h); }
API Node* fo_clone(Node* n) { return n->clone(); }
API void fo_free(Node* n) { delete n; }

// ---- Wave::render (src/wave.rs:441-466): out is [channels][length], length = round(duration * sr)
static void render_impl(Node* node, size_t length, float* out, size_t out_stride) {
  const int no = node->outputs();
  std::vector<float> buf((size_t)no * B, 0.0f);
  size_t i = 0;
  while (i < length) {
    int n = (int)std::min<size_t>(length - i, B);
    node->process(n, nullptr, buf.data());
    for (int c = 0; c < no; c++) memcpy(out + c * out_stride + i, buf.data() + c * B, sizeof(float) * n);
    i += n;
  }
}
API int64_t fo_render_length(double sr, double duration) { return (int64_t)round(duration * sr); }
API void fo_render(Node* node, double sr, double duration, float* out) {
  assert(node->inputs() == 0);
  node->set_sample_rate(sr);
  size_t length = (size_t)round(duration * sr);
  render_impl(node, length, out, length);
}
// Wave::filter (src/wave.rs:518-565): in is [inputs][in_len], out is [outputs][total_len]
API void fo_filter(Node* node, double sr, const float* in, int64_t in_len, int64_t total_len, float* out) {
  node->set_sample_rate(sr);
  const int ni = node->inputs(), no = node->outputs();
  std::vector<float> ib((size_t)std::max(1, ni) * B, 0.0f), ob((size_t)no * B, 0.0f);
  int64_t input_length = std::min(total_len, in_len);
  int64_t i = 0;
  while (i < total_len) {
    bool from_wave = i < input_length;
    int n = (int)std::min<int64_t>((from_wave ? input_length : total_len) - i, B);
    if (from_wave) { for (int c = 0; c < ni; c++) for (int j = 0; j < n; j++) ib[c * B + j] = in[c * in_len + i + j]; }
    else std::fill(ib.begin(), ib.end(), 0.0f);
    node->process(n, ib.data(), ob.data());
    for (int c = 0; c < no; c++) memcpy(out + c * total_len + i, ob.data() + c * B, sizeof(float) * n);
    i += n;
  }
}
// continue rendering without touching the sample rate (n samples, block 64), used for process()-granularity checks
API void fo_process_many(Node* node, int64_t n, const float* in, float* out) {
  const int ni = node->inputs(), no = node->outputs();
  std::vector<float> ib((size_t)std::max(1, ni) * B, 0.0f), ob((size_t)std::max(1, no) * B, 0.0f);
  int64_t i = 0;
  while (i < n) {
    int m = (int)std::min<int64_t>(n - i, B);
    for (int c = 0; c < ni; c++) for (int j = 0; j < m; j++) ib[c * B + j] = in[c * n + i + j];
    node->process(m, ib.data(), ob.data());
    for (int c = 0; c < no; c++) memcpy(out + c * n + i, ob.data() + c * B, sizeof(float) * m);
    i += m;
  }
}

// ---- Net (src/net.rs). Node ids are vertex indices (the oracle never removes vertices).
API Node* fo_net_new(int inputs, int outputs) { return new Net(inputs, outputs); }
API Node* fo_net_wrap(Node* unit) { return Net::wrap(unit); }
API int fo_net_push(Node* net, Node* unit) { return static_cast<Net*>(net)->push(unit); }
API int fo_net_chain(Node* net, Node* unit) { return static_cast<Net*>(net)->chain(unit); }
API void fo_net_connect(Node* net, int s, int sp, int t, int tp) { static_cast<Net*>(net)->connect(s, sp, t, tp); }
API void fo_net_connect_input(Node* net, int gi, int t, int tp) { static_cast<Net*>(net)->connect_input(gi, t, tp); }
API void fo_net_connect_output(Node* net, int s, int sp, int go) { static_cast<Net*>(net)->connect_output(s, sp, go); }
API void fo_net_pipe_input(Node* net, int t) { static_cast<Net*>(net)->pipe_input(t); }
API void fo_net_pipe_output(Node* net, int s) { static_cast<Net*>(net)->pipe_output(s); }
API void fo_net_pipe_all(Node* net, int s, int t) { static_cast<Net*>(net)->pipe_all(s, t); }
API void fo_net_pass_through(Node* net, int gi, int go) { static_cast<Net*>(net)->pass_through(gi, go); }
API void fo_net_crossfade(Node* net, int node, int fade, float fade_time, Node* unit) { static_cast<Net*>(net)->crossfade(node, fade, fade_time, unit); }   // Net::crossfade (src/net.rs:480-504)
API int fo_net_size(Node* net) { return (int)static_cast<Net*>(net)->vertex.size(); }
API int fo_net_has_cycle(Node* net) { Net* n = static_cast<Net*>(net); if (!n->ordered) n->determine_order(); return n->cycle ? 1 : 0; }
API int fo_net_order(Node* net, int* out) { Net* n = static_cast<Net*>(net); if (!n->ordered) n->determine_order(); for (size_t i = 0; i < n->order.size(); i++) out[i] = n->order[i]; return (int)n->order.size(); }
// algebra: op 0 bus(&), 1 pipe(>>), 2 stack(|), 3 branch(^), 4 sum(+), 5 product(*), 6 sub(-)
API Node* fo_net_combine(int op, Node* a, Node* b) {
  Net* x = static_cast<Net*>(a); Net* y = static_cast<Net*>(b);
  switch (op) { case 0: return Net::bus(x, y); case 1: return Net::pipe(x, y); case 2: return Net::stack(x, y); case 3: return Net::branch(x, y);
    case 4: return Net::binary(x, y, OP_ADD); case 5: return Net::binary(x, y, OP_MUL); default: return Net::binary(x, y, OP_SUB); }
}

// ---- voice-bank CPU baseline: V independent units, block-64 `process`, contiguous shards over threads;
// per-voice outputs [V][channels][n] (out may be null) and/or sequential index-order mix [channels][n].
API void fo_bank_render(Node** voices, int64_t nvoices, double sr, int64_t n, const float* in /*[inputs][n] shared*/, float* out, float* mix, int nthreads) {
  if (nvoices == 0) return;
  const int no = voices[0]->outputs(), ni = voices[0]->inputs();
  for (int64_t v = 0; v < nvoices; v++) voices[v]->set_sample_rate(sr);
  if (nthreads < 1) nthreads = 1;
  std::vector<std::vector<float>> partial;
  if (mix) partial.assign(nthreads, std::vector<float>((size_t)no * n, 0.0f));
  auto work = [&](int t) {
    int64_t v0 = nvoices * t / nthreads, v1 = nvoices * (t + 1) / nthreads;
    std::vector<float> ib((size_t)std::max(1, ni) * B, 0.0f), ob((size_t)no * B, 0.0f);
    for (int64_t i = 0; i < n; i += B) {
      int m = (int)std::min<int64_t>(n - i, B);
      for (int c = 0; c < ni; c++) for (int j = 0; j < m; j++) ib[c * B + j] = in[c * n + i + j];
      for (int64_t v = v0; v < v1; v++) {
        voices[v]->process(m, ib.data(), ob.data());
        for (int c = 0; c < no; c++) {
          if (out) memcpy(out + ((size_t)v * no + c) * n + i, ob.data() + c * B, sizeof(float) * m);
          if (mix) { float* p = partial[t].data() + (size_t)c * n + i; for (int j = 0; j < m; j++) p[j] += ob[c * B + j]; }
        }
      }
    }
  };
  std::vector<std::thread> th;
  for (int t = 1; t < nthreads; t++) th.emplace_back(work, t);
  work(0);
  for (auto& x : th) x.join();
  if (mix) {
    for (size_t k = 0; k < (size_t)no * n; k++) { float s = partial[0][k]; for (int t = 1; t < nthreads; t++) s += partial[t][k]; mix[k] = s; }
  }
}

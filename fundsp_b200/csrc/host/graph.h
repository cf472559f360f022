// fundsp_b200 host graph: construction-time mirror of the reference's AudioNode tree.
//
// The reference builds a typed tree of nodes (`An<X>`, src/combinator.rs:178) whose constructors thread a
// deterministic hash through the tree (`ping`, src/audionode.rs:156-161 and every combinator `new`), apply
// `Setting`s (src/setting.rs) and compute coefficients in `set_sample_rate`. This file keeps exactly that
// construction-time behaviour on the host and *lowers* a tree to what the GPU needs:
//   - a type expression (`sig`) naming the fused device program in csrc/dsp/nodes.cuh,
//   - per-voice parameter words (P), per-voice initial state words (S), class-uniform words (U) and
//     delay-line lengths, all in depth-first left-to-right order (the order Loader consumes them).
// No audio is processed here; the product has no CPU DSP path.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

namespace fdsp {
namespace host {

constexpr double DEFAULT_SR = 44100.0;  // src/lib.rs:42

// ---- hashing (src/math.rs:569-576, 632-658)
inline double rnd1(uint64_t x) {
  x ^= 0x5555555555555555ull;
  x *= 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  x ^= x >> 31;
  return (double)(x >> 11) * (1.0 / 9007199254740992.0);
}
struct AttoHash {
  uint64_t state;
  explicit AttoHash(uint64_t s = 0) : state(s) {}
  AttoHash hash(uint64_t data) const { return AttoHash((((state << 5) | (state >> 59)) ^ data) * 0x517cc1b727220a95ull); }
};

// ---- settings (src/setting.rs:14-62); same numbering as the C ABI (include/fundsp_b200.h)
enum ParamKind { P_NULL = 0, P_CENTER, P_CENTER_Q, P_CENTER_Q_GAIN, P_VALUE, P_COEFFICIENT, P_BIQUAD, P_DELAY, P_TIME,
                 P_ROUGHNESS, P_VARIABILITY, P_PAN, P_ATTACK_RELEASE, P_PHASE, P_SEED, P_INTERVAL };
struct Address { int type; uint64_t value; };  // 1 Index, 2 Node
struct Setting {
  int kind = P_NULL; float v[5] = {0, 0, 0, 0, 0}; uint64_t seed = 0; std::vector<Address> address;
  Address direction() const { return address.empty() ? Address{0, 0} : address[0]; }
  Setting peel() const { Setting s = *this; if (!s.address.empty()) s.address.erase(s.address.begin()); return s; }
};

inline uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

// ---- Shared (src/shared.rs:47-81): a 32-bit cell that any thread sets and reads with relaxed atomics, like the AtomicU32 behind a
// Rust Shared. Reference counted: the creator's handle and every node (and bank) that uses the cell hold one reference each, as an
// Arc clone does. `external`: the cell is memory the caller owns (the AtomicU32 of a Rust Shared); `release(user)` runs when the last
// reference goes, so the owner can keep the memory alive until then (the Rust binding passes a leaked Arc clone and drops it there).
struct SharedCell {
  uint32_t own = 0; uint32_t* cell; int refs = 1;
  void (*release)(void*) = nullptr; void* user = nullptr;
  explicit SharedCell(float v) : own(f2u(v)), cell(&own) {}
  SharedCell(uint32_t* external, void (*rel)(void*), void* u) : cell(external), release(rel), user(u) {}
  ~SharedCell() { if (release) release(user); }
  SharedCell(const SharedCell&) = delete;
  SharedCell& operator=(const SharedCell&) = delete;
  uint32_t get() const { return __atomic_load_n(cell, __ATOMIC_RELAXED); }
  void set(uint32_t w) { __atomic_store_n(cell, w, __ATOMIC_RELAXED); }
  SharedCell* ref() { __atomic_add_fetch(&refs, 1, __ATOMIC_RELAXED); return this; }
  void unref() { if (__atomic_sub_fetch(&refs, 1, __ATOMIC_ACQ_REL) == 0) delete this; }
};
struct SharedRef {   // one counted reference
  SharedCell* c = nullptr;
  SharedRef() {}
  explicit SharedRef(SharedCell* x) : c(x ? x->ref() : nullptr) {}
  SharedRef(const SharedRef& o) : c(o.c ? o.c->ref() : nullptr) {}
  SharedRef& operator=(const SharedRef& o) { if (this != &o) { SharedCell* n = o.c ? o.c->ref() : nullptr; if (c) c->unref(); c = n; } return *this; }
  ~SharedRef() { if (c) c->unref(); }
};
// A word of a lowered voice that is tied to a Shared: the parameter word of a reader (Var, VarFn input), or the state word in which a
// writer (Monitor, Timer) leaves the value it stores.
enum SharedUseKind { SH_READ = 0, SH_MONITOR = 1, SH_TIMER = 2 };
struct SharedUse { uint32_t word; SharedCell* cell; int kind; };

struct HNode;

struct Lowering {
  std::vector<uint32_t> P, S, U;   // words in DFS order
  std::vector<uint32_t> dlen;      // delay-line lengths (floats per voice) in DFS order
  uint32_t extraU = 0;             // uniform words beyond the nodes' static NU (e.g. a Convolver's impulse response)
  uint32_t extraP = 0;             // per-voice parameter words beyond the static NP (an envelope's sampled closure values)
  uint32_t conv_K = 0, conv_off = 0;   // last Convolver lowered: taps, and the index of its header (K, ring length, then K coefficient words) in U
  // [begin, end) of state words / of `dlen` entries that AudioUnit::reset leaves ALONE where the reference's reset does (Reverb::reset keeps
  // its pre-delay allpasses, src/reverb.rs:215-228; Limiter::reset keeps its follower, src/dynamics.rs:181-195): Bank::reset skips them
  std::vector<std::pair<uint32_t, uint32_t>> keepS, keepD;
  // (state word, value) pairs where what reset() restores differs from the state a freshly built unit starts from (Adaptive's level
  // estimate: 0.0 after Adaptive::new, 1e-3 after reset, src/shape.rs:173-196). Every other word resets to its lowered value.
  std::vector<std::pair<uint32_t, uint32_t>> resetS;
  // [begin, end) of state words that the Setting just applied to the node wrote (a System's target values): Bank::set copies them into
  // the running state, where the device reads them at the next launch
  std::vector<std::pair<uint32_t, uint32_t>> liveS;
  std::vector<SharedUse> shared;   // Shared readers and writers in evaluation order
  // writers are refused inside units that run on a clock of their own (events, slots, crossfades): the order of their stores is not the bank's
  void no_writers_since(size_t k, const char* where) { for (; k < shared.size(); k++) if (shared[k].kind != SH_READ) { fail(std::string("monitor / timer writing a Shared inside ") + where + " is not supported"); return; } }
  bool ok = true; std::string why; // set when a node has no device lowering
  // where one node's words sit in its voice's lowering (Bank::set_voices): the combinators a Setting walks through (reach_setting, and a
  // sequencer event) lower their children through sub(), which records the [begin, end) of P and S that `mark` lowers
  const HNode* mark = nullptr; bool marked = false; uint32_t mark_p[2] = {0, 0}, mark_s[2] = {0, 0};
  inline void sub(const HNode* n);
  void p(float f) { P.push_back(f2u(f)); }
  void s(float f) { S.push_back(f2u(f)); }
  void su(uint32_t u) { S.push_back(u); }
  // an f64 word pair, low word first (the prelude64 nodes)
  void p64(double d) { uint64_t u; memcpy(&u, &d, 8); P.push_back((uint32_t)u); P.push_back((uint32_t)(u >> 32)); }
  void s64(double d) { uint64_t u; memcpy(&u, &d, 8); S.push_back((uint32_t)u); S.push_back((uint32_t)(u >> 32)); }
  void s_reset(float now, float on_reset) { resetS.emplace_back((uint32_t)S.size(), f2u(on_reset)); s(now); }
  std::vector<uint32_t> reset_image() const { std::vector<uint32_t> r = S; for (auto& w : resetS) if (w.first < r.size()) r[w.first] = w.second; return r; }
  void fail(const std::string& w) { if (ok) { ok = false; why = w; } }
};

struct HNode {
  virtual ~HNode() {}
  virtual int inputs() const = 0;
  virtual int outputs() const = 0;
  virtual uint64_t id() const = 0;
  virtual void reset() {}
  virtual void set_sample_rate(double) {}
  virtual void set(const Setting&) {}
  virtual void set_hash(uint64_t) {}
  virtual AttoHash ping(bool probe, AttoHash hash);
  virtual HNode* clone() const = 0;
  virtual void sig(std::string& out) const = 0;
  virtual void lower(Lowering& l) const = 0;
  void ctor_ping() { AttoHash h = ping(true, AttoHash(id())); ping(false, h); }
  static std::vector<uint64_t>*& ping_trace();
};
inline void Lowering::sub(const HNode* n) {
  if (n != mark) { n->lower(*this); return; }
  mark_p[0] = (uint32_t)P.size(); mark_s[0] = (uint32_t)S.size();
  n->lower(*this);
  mark_p[1] = (uint32_t)P.size(); mark_s[1] = (uint32_t)S.size(); marked = true;
}

// Where a Setting goes inside `n`, as the combinators' own set() forwards it: an Index peels one step into a binary combinator or a Multi;
// Unop and Thru pass the setting on unchanged; Feedback keeps it. Returns the node at which that walk ends, with *s as it arrives there
// (`hops`: the child taken at each step), or null when the address leads nowhere (the combinator ignores the setting).
HNode* reach_setting(HNode* n, Setting* s, std::vector<int>* hops);
// The node that `voice->set(s)` changes, when nothing else changes: reach_setting, entered through a sequencer event (whose set() only
// forwards to its unit), with *s as that node receives it. *ignored: the setting leads nowhere. Null as well when the walk ends at a node
// whose set() does more than change its own words: a System (it also writes its targets' values into the running state), a Net, a Slot,
// a crossfading vertex.
HNode* setting_leaf(HNode* voice, Setting* s, bool* ignored);

// The nodes whose set() the device computes (the targets of update(), nodes.cuh UpdTarget, and of Bank::set_voices_device), with what
// their set() reads and writes. kind: 0 FixedSvf (mode 0-8), 1 the fixed ButterLowpass, 3 the fixed Biquad, 4 Lowpole, 5 Highpole,
// 6 DCBlock (the fixed one-poles), 7 Constant (nch channels), 8 Panner<U1>. v: (cutoff, q, gain), (cutoff), (a1, a2, b0, b1, b2),
// (cutoff), (cutoff), (cutoff), (value), (pan). sr: the node's own sample rate.
struct Controls { int kind = -1, mode = 0, nch = 0; float sr = 0.0f; float v[5] = {0, 0, 0, 0, 0}; };
bool read_controls(HNode* n, Controls* c);                 // false: n is none of those nodes
int controls_taken(int kind, int setting);                 // the leading values of v a setting of that kind writes (0: the node ignores it)
Setting controls_setting(const Controls& c);               // the setting that gives such a node the values c.v (with its own sample rate)
bool setting_ignored(const HNode* n, const Setting& s);    // n.set(s) leaves every word n lowers as it was

// ---- builders (one per primitive; composites consume their children)
HNode* mk_constant(int n, const float* v);
HNode* mk_pass();
HNode* mk_monitor();   // Monitor ID 56: pass-through in the audio path
HNode* mk_multipass(int n);
HNode* mk_sink(int n);
HNode* mk_split(int n);
HNode* mk_multisplit(int m, int n);
HNode* mk_join(int n);
HNode* mk_multijoin(int m, int n);
HNode* mk_reverse(int n);
HNode* mk_sine();
HNode* mk_wavesynth(int kind, int outputs);
HNode* mk_noise();
HNode* mk_fixed_svf(int mode, float cutoff, float q, float gain);
HNode* mk_svf(int mode, float cutoff, float q, float gain);
// prelude64: Sine<f64> (ID 21), FixedSvf<f64, M> (ID 43), Svf<f64, M> (ID 36); f32 arguments widened with F::from_f32
HNode* mk_sine64();
HNode* mk_fixed_svf64(int mode, float cutoff, float q, float gain);
HNode* mk_svf64(int mode, float cutoff, float q, float gain);
// Biquad<f64> ID 15, ButterLowpass<f64, U1|U2> ID 16, Resonator<f64, U1|U3> ID 17; the one-pole family as mk_onepole with F = f64
HNode* mk_biquad64(float a1, float a2, float b0, float b1, float b2);
HNode* mk_butterpass64(float cutoff, int nin);
HNode* mk_resonator64(float center, float q, int nin);
HNode* mk_onepole64(int kind, float param, int inputs);
HNode* mk_biquad(float a1, float a2, float b0, float b1, float b2);
HNode* mk_biquad_bank();
HNode* mk_butterpass(float cutoff, int nin);
HNode* mk_resonator(float center, float q, int nin);
HNode* mk_moog(float cutoff, float q, int nin);
HNode* mk_fir(int n, const float* w);
HNode* mk_tick(int n);
HNode* mk_delay(double t);
HNode* mk_allnest(float coefficient, HNode* x, int nin);
HNode* mk_phase_osc(int kind);                      // 0 ramp, 1 poly_saw, 2 poly_square, 3 poly_pulse
HNode* mk_reverb3(double time, double diffusion, HNode* filter);   // Reverb<F> ID 85; consumes `filter` (1 -> 1)
HNode* mk_var(float value);
// Shared controls (src/shared.rs, src/dynamics.rs:441-520). Each node takes a reference to the cell.
HNode* mk_var_shared(SharedCell* s);                                  // Var ID 68: the cell's value, fixed for one call
HNode* mk_monitor_shared(SharedCell* s, int kind, double timescale);  // Monitor ID 56: passes through, stores the meter level (kind as mk_meter)
HNode* mk_timer(SharedCell* s);
// VarFn ID 70: the closure (text, as mk_closure's, one parameter |x|) of the cell's value, with 1-8 outputs; null with the reason in `err`
HNode* mk_var_fn(SharedCell* s, int outputs, const char* text, int ncaptures, const char* const* names, const float* values, std::string& err);                                       // Timer ID 57: stores the stream time; sets the cell to 0 now
HNode* mk_nl_biquad(int fb, int mode, int shape, float p0, float p1, int inputs, float center, float q, float gain);  // IDs 88-91
HNode* mk_phase_synth(int kind);                                     // PhaseSynth ID 35
HNode* mk_pulse();                                                   // PulseWave ID 44
HNode* mk_mixer(int inputs, int outputs, const float* matrix);       // Mixer ID 84, matrix[output][input]
HNode* mk_rotate(float angle, float gain);                           // rotate(): 2x2 Mixer
HNode* mk_meter(int kind, double timescale);                         // MeterNode ID 61: kind 0 Sample, 1 Peak, 2 Rms
HNode* mk_playwave(const float* samples, uint64_t length, uint64_t start, uint64_t end, int64_t loop_point);  // WavePlayer ID 65
HNode* mk_resample(HNode* x);                                        // Resample<X> ID 69; consumes the generator
HNode* mk_limiter(int channels, float attack, float release);       // Limiter<N> ID 25
HNode* mk_event(HNode* x, double start, double end, int fade_ease, double fade_in, double fade_out);  // one Sequencer event (ID 64) as a voice; consumes x
bool event_edit(HNode* n, double end_time, double fade_out);         // false when n is not an event
bool event_times(const HNode* n, double* start, double* end);
HNode* mk_event_loop(HNode* x, double start, double end, int fade_ease, double fade_in, double fade_out, double loop_seconds);  // an event of a ReplayMode::Loop(loop_seconds) sequencer
bool event_loop(const HNode* n, double* loop_seconds);               // false when n is not an event; 0 = the event's sequencer does not loop
bool event_set_clock(HNode* n, double time);                         // the sequencer time the event's own clock starts from
// Sequencer::set_sample_rate to a new rate (src/sequencer.rs:750-765) ends in Sequencer::reset, which without a loop resets the unit of every
// event (:720-733): true when n is such an event and `s` differs from its rate. Sequencer::push only re-rates a unit (:369), never resets it.
bool event_rerate_resets(const HNode* n, double s);
// Envelope<F, E, R> (ID 14): `f(t, out[outputs], user)` is the closure E, evaluated ON THE HOST at the reference's sample points when the
// graph is lowered (bank creation, sample-rate change, settings) for t <= horizon seconds; time_f64: F = f64 (else f32)
typedef void (*EnvelopeFn)(double t, double* out, void* user);
HNode* mk_envelope(double interval, int outputs, int time_f64, EnvelopeFn f, void* user, double horizon);
HNode* mk_oversample(HNode* x);                                      // Oversampler ID 51; consumes x
HNode* mk_xfade(HNode* x, HNode* y, int ease, float fade_time);        // a Net vertex fading from x to y (Net::crossfade); consumes both
bool xfade_set_done(HNode* n, bool done);                            // lower the vertex as already arrived at its second unit (what a bank reset restores)
bool xfade_fade(const HNode* n, float* fade_time, float* sr);                              // the f32 fade time and rate the vertex's crossfade runs with
const HNode* xfade_unit(const HNode* n, int which);                  // 0: the unit being faded out, 1: the unit being faded in; null when n is not a crossfading vertex
HNode* mk_slot(HNode* x);                                            // SlotBackend ID 78: a replaceable unit; consumes x
bool slot_arm(HNode* slot, HNode* unit, int instance, int ease, double fade_time);   // consumes unit
bool is_slot(const HNode* n);
bool slot_fade(const HNode* slot, double* fade_time, double* sr);                      // the fade time and rate the slot's crossfade runs with (its parameter words)
HNode* mk_declick(float duration);                                   // Declick ID 23
HNode* mk_chaos(int kind);                                           // 0 Rossler ID 73, 1 Lorenz ID 74
HNode* mk_morph(float cutoff, float q);                               // Morph ID 62
HNode* mk_rez(float bandpass, float cutoff, float q, int inputs);    // Rez ID 75 (bandpass 0 lowrez / 1 bandrez)
HNode* mk_follow(int asymmetric, float attack, float release);        // Follow ID 24 / AFollow ID 29
HNode* mk_shaper(int kind, float p0, float p1);                       // Shaper ID 42: 0 Clip 1 ClipTo 2 Tanh 3 Softsign 4 Crush 5 SoftCrush 6 Atan
// Shaper<Adaptive<S>> ID 42 / nonlinear biquads with an Adaptive shape: `inner` is one of the Shaper kinds 0..6 with its (p0, p1);
// on failure null with the reason in `err`
HNode* mk_shaper_adaptive(double timescale, int inner, float p0, float p1, std::string& err);
HNode* mk_nl_biquad_adaptive(int fb, int mode, double timescale, int inner, float p0, float p1, int inputs, float center, float q, float gain, std::string& err);
HNode* mk_onepole(int kind, float param, int inputs);                  // 0 Lowpole 18, 1 Highpole 47, 2 Allpole 46, 3 DCBlock 22, 4 Pinkpass 26
HNode* mk_convolve(const float* response, int n);                     // Convolver ID 100
HNode* mk_feedback_unit(double delay, HNode* x);                      // FeedbackUnit ID 79                                          // Var ID 68
HNode* mk_dsf(int inputs, float harmonic_spacing, float roughness);
HNode* mk_mls(int bits);
HNode* mk_impulse(int n);
HNode* mk_tap(int ntaps, int linear, float min_delay, float max_delay);
HNode* mk_feedback2(HNode* x, HNode* y, int hadamard);
HNode* mk_pan(float value);
HNode* mk_panner();
HNode* mk_adsr_live(float a, float d, float s, float r);
// closures of the signal or of time, parsed from text (closure.h): kind 0 Map ID 5, 1 Shaper<ShapeFn> ID 42, 2 EnvelopeIn<f32> ID 53, 4 Envelope<f32>
// ID 14 (`interval` seconds for both envelopes; no horizon: the device evaluates the closure at every sample point);
// captures are (name, value) pairs. On failure returns null with the reason in `err` (arity mismatches start with "<what>: arity mismatch").
HNode* mk_closure(int kind, int inputs, int outputs, double interval, const char* text, int ncaptures, const char* const* names, const float* values,
                  std::string& err);
// System<X, F> ID 67 (`update(x, dt, f)`): the closure `|t, dt, x| ..` (text, closure.h CL_UPDATE) sets x's parameters every ~dt seconds;
// consumes x. On failure null with the reason in `err`. A `set` reaching a node the device cannot set is refused when the graph is lowered.
HNode* mk_update(HNode* x, float dt, const char* text, int ncaptures, const char* const* names, const float* values, std::string& err);
HNode* mk_pipe(HNode* x, HNode* y);
HNode* mk_stack(HNode* x, HNode* y);
HNode* mk_branch(HNode* x, HNode* y);
HNode* mk_bus(HNode* x, HNode* y);
HNode* mk_thru(HNode* x);
HNode* mk_binop(int op, HNode* x, HNode* y);
HNode* mk_unop(int kind, float scalar, HNode* x);
HNode* mk_multi(int kind, int op, int n, HNode** nodes);
HNode* mk_feedback(HNode* x, int hadamard);

// ---- Net (src/net.rs:118-146): dynamic DAG of units. Vertex ids are indices (this mirror never removes vertices).
HNode* mk_net(int inputs, int outputs);
bool is_net(const HNode* n);
int net_push(HNode* net, HNode* unit);                                 // Net::push (src/net.rs:204-213): sets the unit's sample rate
bool net_connect(HNode* net, int src, int src_port, int dst, int dst_port);   // Net::connect
bool net_connect_input(HNode* net, int global_in, int dst, int dst_port);     // Net::connect_input
bool net_connect_output(HNode* net, int src, int src_port, int global_out);   // Net::connect_output
bool net_pass_through(HNode* net, int global_in, int global_out);             // Net::pass_through
int net_size(const HNode* net);
// A voice-separable Net: every global output is an adder tree (Binop<Add,Pass,Pass> vertices, as built by Net::bus /
// `&`) over the same sequence of voice vertices. Extracts the voices in leaf order; `tree` receives the canonical
// description ("pairwise" when the tree is the level-wise adjacent pairing, "chain" for a left fold). Pings the net first
// (Net::determine_order, src/net.rs:834-852) so the voices carry the hashes the reference would give them.
bool net_extract_voices(HNode* net, std::vector<HNode*>& voices, std::string& tree, std::string& err, std::vector<int>* vertex_ids = nullptr);

// ---- wavetables (src/wavetable.rs:40-123, 493-623): built once per waveform kind on the host
struct WaveTableHost { std::vector<float> pitch; std::vector<int> off, len; std::vector<float> data; };
const WaveTableHost& global_wavetable(int kind);
const WaveTableHost& device_wavetable(int kind);   // same tables with wrap-around guard samples (the layout the kernels read)

}  // namespace host
}  // namespace fdsp

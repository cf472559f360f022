// fundsp_b200 C ABI (include/fundsp_b200.h): thin, exception-free shell over csrc/host.
#include "../../include/fundsp_b200.h"

#include <cstring>
#include <new>
#include <algorithm>
#include <string>
#include <vector>

#include "host/bank.h"
#include "host/closure.h"
#include "host/group.h"
#include "host/wavfile.h"

using namespace fdsp::host;

struct fdsp_node { HNode* n; };
struct fdsp_bank { Bank b; };

namespace {
thread_local std::string g_err;
int fail(int code, const std::string& msg) { g_err = msg; return code; }
fdsp_node* wrap(HNode* n, const char* what) {
  if (!n) { g_err = std::string(what) + ": arity mismatch or invalid argument (the reference rejects this at compile time)"; return nullptr; }
  fdsp_node* h = new (std::nothrow) fdsp_node{n};
  if (!h) { delete n; g_err = std::string(what) + ": out of memory"; }
  return h;
}
HNode* take(fdsp_node* h) {  // consume a handle
  if (!h) return nullptr;
  HNode* n = h->n; delete h; return n;
}
// Runtime messages carry their status as a leading tag (csrc/host/bank.h): "#U " unsupported, "#A " argument, "#N " no free slot.
char tag_of(const std::string& e) { return e.size() > 3 && e[0] == '#' && e[2] == ' ' ? e[1] : 0; }
int status(const std::string& e, int untagged = FDSP_ERR_CUDA) {
  if (e.empty()) return FDSP_OK;
  const char t = tag_of(e);
  if (t == 'U') return fail(FDSP_ERR_UNSUPPORTED, e.substr(3));
  if (t == 'A' || t == 'N') return fail(FDSP_ERR_ARG, e.substr(3));
  return fail(e.find("no device lowering") != std::string::npos ? FDSP_ERR_UNSUPPORTED : untagged, e);
}
}  // namespace

#define API extern "C" __attribute__((visibility("default")))

API const char* fdsp_version(void) { return "fundsp_b200 0.1.0 (sm_90a; mirrors fundsp 0.23.0 hot path)"; }
API const char* fdsp_last_error(void) { return g_err.c_str(); }
API int fdsp_device_count(void) { int n = 0; return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0; }

API fdsp_node* fdsp_constant(int n, const float* v) { return (n < 1 || !v) ? wrap(nullptr, "constant") : wrap(mk_constant(n, v), "constant"); }
API fdsp_node* fdsp_pass(void) { return wrap(mk_pass(), "pass"); }
API fdsp_node* fdsp_multipass(int n) { return wrap(n < 0 ? nullptr : mk_multipass(n), "multipass"); }
API fdsp_node* fdsp_sink(int n) { return wrap(n < 1 ? nullptr : mk_sink(n), "sink"); }
API fdsp_node* fdsp_split(int n) { return wrap(n < 1 ? nullptr : mk_split(n), "split"); }
API fdsp_node* fdsp_multisplit(int m, int n) { return wrap((m < 1 || n < 1) ? nullptr : mk_multisplit(m, n), "multisplit"); }
API fdsp_node* fdsp_join(int n) { return wrap(n < 1 ? nullptr : mk_join(n), "join"); }
API fdsp_node* fdsp_multijoin(int m, int n) { return wrap((m < 1 || n < 1) ? nullptr : mk_multijoin(m, n), "multijoin"); }
API fdsp_node* fdsp_reverse(int n) { return wrap(n < 1 ? nullptr : mk_reverse(n), "reverse"); }
API fdsp_node* fdsp_sine(void) { return wrap(mk_sine(), "sine"); }
API fdsp_node* fdsp_wavesynth(int table, int outputs) { return wrap(mk_wavesynth(table, outputs), "wavesynth"); }
API fdsp_node* fdsp_noise(void) { return wrap(mk_noise(), "noise"); }
API fdsp_node* fdsp_fixed_svf(int mode, float c, float q, float g) { return wrap(mk_fixed_svf(mode, c, q, g), "fixed_svf"); }
API fdsp_node* fdsp_svf(int mode, float c, float q, float g) { return wrap(mk_svf(mode, c, q, g), "svf"); }
API fdsp_node* fdsp_sine_f64(void) { return wrap(mk_sine64(), "sine_f64"); }
API fdsp_node* fdsp_fixed_svf_f64(int mode, float c, float q, float g) { return wrap(mk_fixed_svf64(mode, c, q, g), "fixed_svf_f64"); }
API fdsp_node* fdsp_svf_f64(int mode, float c, float q, float g) { return wrap(mk_svf64(mode, c, q, g), "svf_f64"); }
API fdsp_node* fdsp_biquad_f64(float a1, float a2, float b0, float b1, float b2) { return wrap(mk_biquad64(a1, a2, b0, b1, b2), "biquad_f64"); }
API fdsp_node* fdsp_butterpass_f64(float c, int nin) { return wrap(mk_butterpass64(c, nin), "butterpass_f64"); }
API fdsp_node* fdsp_resonator_f64(float c, float q, int nin) { return wrap(mk_resonator64(c, q, nin), "resonator_f64"); }
API fdsp_node* fdsp_onepole_f64(int kind, float param, int inputs) { return wrap(mk_onepole64(kind, param, inputs), "onepole_f64"); }
API fdsp_node* fdsp_biquad(float a1, float a2, float b0, float b1, float b2) { return wrap(mk_biquad(a1, a2, b0, b1, b2), "biquad"); }
API fdsp_node* fdsp_biquad_bank(void) { return wrap(mk_biquad_bank(), "biquad_bank"); }
API fdsp_node* fdsp_butterpass(float c, int nin) { return wrap((nin < 1 || nin > 2) ? nullptr : mk_butterpass(c, nin), "butterpass"); }
API fdsp_node* fdsp_resonator(float c, float q, int nin) { return wrap((nin != 1 && nin != 3) ? nullptr : mk_resonator(c, q, nin), "resonator"); }
API fdsp_node* fdsp_moog(float c, float q, int nin) { return wrap(mk_moog(c, q, nin), "moog"); }
API fdsp_node* fdsp_fir(int n, const float* w) { return wrap((n < 1 || !w) ? nullptr : mk_fir(n, w), "fir"); }
API fdsp_node* fdsp_tick(int n) { return wrap(n < 1 ? nullptr : mk_tick(n), "tick"); }
API fdsp_node* fdsp_delay(double t) { return wrap(mk_delay(t), "delay"); }
API fdsp_node* fdsp_allnest(float c, fdsp_node* x, int nin) { return wrap(mk_allnest(c, take(x), nin), "allnest"); }
API fdsp_node* fdsp_phase_osc(int kind) { return wrap(mk_phase_osc(kind), "phase_osc"); }
API fdsp_node* fdsp_reverb3(double time, double diffusion, fdsp_node* filter) { return wrap(mk_reverb3(time, diffusion, take(filter)), "reverb3"); }
API fdsp_node* fdsp_feedback_unit(double delay, fdsp_node* x) { return wrap(mk_feedback_unit(delay, take(x)), "feedback_unit"); }
API fdsp_node* fdsp_convolve(const float* response, int n) { return wrap(mk_convolve(response, n), "convolve"); }
API fdsp_node* fdsp_onepole(int kind, float param, int inputs) { return wrap(mk_onepole(kind, param, inputs), "onepole"); }
API fdsp_node* fdsp_shaper(int kind, float p0, float p1) { return wrap(mk_shaper(kind, p0, p1), "shaper"); }
API fdsp_node* fdsp_follow(int asymmetric, float attack, float release) { return wrap(mk_follow(asymmetric, attack, release), "follow"); }
API fdsp_node* fdsp_morph(float cutoff, float q) { return wrap(mk_morph(cutoff, q), "morph"); }
API fdsp_node* fdsp_rez(float bandpass, float cutoff, float q, int inputs) { return wrap(mk_rez(bandpass, cutoff, q, inputs), "rez"); }
API fdsp_node* fdsp_chaos(int kind) { return wrap(mk_chaos(kind), "chaos"); }
API fdsp_node* fdsp_declick(float duration) { return wrap(mk_declick(duration), "declick"); }
API fdsp_node* fdsp_slot(fdsp_node* unit) { return wrap(mk_slot(take(unit)), "slot"); }
API fdsp_node* fdsp_oversample(fdsp_node* x) { return wrap(mk_oversample(take(x)), "oversample"); }
API fdsp_node* fdsp_monitor(void) { return wrap(mk_monitor(), "monitor"); }
API fdsp_node* fdsp_envelope(double interval, int outputs, int time_f64, fdsp_envelope_fn f, void* user, double horizon) { return wrap(mk_envelope(interval, outputs, time_f64, (EnvelopeFn)f, user, horizon), "envelope"); }
API fdsp_node* fdsp_event(fdsp_node* x, double start, double end, int fade_ease, double fade_in, double fade_out) { return wrap(mk_event(take(x), start, end, fade_ease, fade_in, fade_out), "event"); }
API fdsp_node* fdsp_event_loop(fdsp_node* x, double start, double end, int fade_ease, double fade_in, double fade_out, double loop_seconds) { return wrap(mk_event_loop(take(x), start, end, fade_ease, fade_in, fade_out, loop_seconds), "event_loop"); }
API fdsp_node* fdsp_limiter(int channels, float attack, float release) { return wrap(mk_limiter(channels, attack, release), "limiter"); }
API fdsp_node* fdsp_meter(int kind, double timescale) { return wrap(mk_meter(kind, timescale), "meter"); }
API fdsp_node* fdsp_playwave(const float* samples, uint64_t length, uint64_t start, uint64_t end, int64_t loop_point) { return wrap(mk_playwave(samples, length, start, end, loop_point), "playwave"); }
API fdsp_node* fdsp_resample(fdsp_node* x) { return wrap(mk_resample(take(x)), "resample"); }
API fdsp_node* fdsp_phase_synth(int kind) { return wrap(mk_phase_synth(kind), "phase_synth"); }
API fdsp_node* fdsp_pulse(void) { return wrap(mk_pulse(), "pulse"); }
API fdsp_node* fdsp_mixer(int inputs, int outputs, const float* matrix) { return wrap(mk_mixer(inputs, outputs, matrix), "mixer"); }
API fdsp_node* fdsp_rotate(float angle, float gain) { return wrap(mk_rotate(angle, gain), "rotate"); }
API fdsp_node* fdsp_nl_biquad(int fb, int mode, int shape, float p0, float p1, int inputs, float center, float q, float gain) {
  return wrap(mk_nl_biquad(fb, mode, shape, p0, p1, inputs, center, q, gain), "nl_biquad");
}
API fdsp_node* fdsp_var(float value) { return wrap(mk_var(value), "var"); }
API fdsp_node* fdsp_dsf(int inputs, float spacing, float roughness) { return wrap(mk_dsf(inputs, spacing, roughness), "dsf"); }
API fdsp_node* fdsp_mls(int bits) { return wrap(mk_mls(bits), "mls"); }
API fdsp_node* fdsp_impulse(int n) { return wrap(mk_impulse(n), "impulse"); }
API fdsp_node* fdsp_tap(int ntaps, int linear, float mn, float mx) { return wrap(mk_tap(ntaps, linear, mn, mx), "tap"); }
API fdsp_node* fdsp_feedback2(fdsp_node* x, fdsp_node* y, int hadamard) { return wrap(mk_feedback2(take(x), take(y), hadamard), "feedback2"); }
API fdsp_node* fdsp_pan(float v) { return wrap(mk_pan(v), "pan"); }
API fdsp_node* fdsp_panner(void) { return wrap(mk_panner(), "panner"); }
API fdsp_node* fdsp_adsr_live(float a, float d, float s, float r) { return wrap(mk_adsr_live(a, d, s, r), "adsr_live"); }
namespace {
fdsp_node* closure_node(int kind, int inputs, int outputs, double interval, const char* closure, int nc, const char* const* names, const float* values) {
  std::string e;
  HNode* n = mk_closure(kind, inputs, outputs, interval, closure, nc, names, values, e);
  if (!n) { g_err = e; return nullptr; }
  return wrap(n, "closure");
}
}  // namespace
API fdsp_node* fdsp_map(int inputs, int outputs, const char* closure, int ncaptures, const char* const* names, const float* values) {
  return closure_node(CL_MAP, inputs, outputs, 0.0, closure, ncaptures, names, values);
}
API fdsp_node* fdsp_shape_fn(const char* closure, int ncaptures, const char* const* names, const float* values) {
  return closure_node(CL_SHAPE_FN, 1, 1, 0.0, closure, ncaptures, names, values);
}
API fdsp_node* fdsp_envelope_in(double interval, int inputs, int outputs, const char* closure, int ncaptures, const char* const* names, const float* values) {
  return closure_node(CL_ENVELOPE_IN, inputs, outputs, interval, closure, ncaptures, names, values);
}
API fdsp_node* fdsp_shaper_adaptive(double timescale, int inner_kind, float p0, float p1) {
  std::string e;
  HNode* n = mk_shaper_adaptive(timescale, inner_kind, p0, p1, e);
  if (!n) { g_err = "shaper_adaptive: " + e; return nullptr; }
  return wrap(n, "shaper_adaptive");
}
API fdsp_node* fdsp_nl_biquad_adaptive(int fb, int mode, double timescale, int inner_kind, float p0, float p1, int inputs, float center, float q, float gain) {
  std::string e;
  HNode* n = mk_nl_biquad_adaptive(fb, mode, timescale, inner_kind, p0, p1, inputs, center, q, gain, e);
  if (!n) { g_err = "nl_biquad_adaptive: " + e; return nullptr; }
  return wrap(n, "nl_biquad_adaptive");
}
API fdsp_node* fdsp_pipe(fdsp_node* x, fdsp_node* y) { return wrap(mk_pipe(take(x), take(y)), "pipe (>>)"); }
API fdsp_node* fdsp_stack(fdsp_node* x, fdsp_node* y) { return wrap(mk_stack(take(x), take(y)), "stack (|)"); }
API fdsp_node* fdsp_branch(fdsp_node* x, fdsp_node* y) { return wrap(mk_branch(take(x), take(y)), "branch (^)"); }
API fdsp_node* fdsp_bus(fdsp_node* x, fdsp_node* y) { return wrap(mk_bus(take(x), take(y)), "bus (&)"); }
API fdsp_node* fdsp_thru(fdsp_node* x) { return wrap(mk_thru(take(x)), "thru (!)"); }
API fdsp_node* fdsp_binop(int op, fdsp_node* x, fdsp_node* y) { return wrap(mk_binop(op, take(x), take(y)), "binop"); }
API fdsp_node* fdsp_unop(int kind, float s, fdsp_node* x) { return wrap(mk_unop(kind, s, take(x)), "unop"); }
API fdsp_node* fdsp_multi(int kind, int op, int n, fdsp_node* const* nodes) {
  if (n < 1 || !nodes) return wrap(nullptr, "multi");
  std::vector<HNode*> v;
  for (int i = 0; i < n; i++) v.push_back(take(nodes[i]));
  return wrap(mk_multi(kind, op, n, v.data()), "multi");
}
API fdsp_node* fdsp_feedback(fdsp_node* x, int hadamard) { return wrap(mk_feedback(take(x), hadamard), "feedback"); }

API fdsp_node* fdsp_net_new(int inputs, int outputs) { return wrap(mk_net(inputs, outputs), "net_new"); }
API int fdsp_net_push(fdsp_node* net, fdsp_node* unit) {
  if (!net || !unit || !is_net(net->n)) { if (unit) fdsp_node_free(unit); return fail(FDSP_ERR_ARG, "net_push: bad arguments") * -1; }
  return net_push(net->n, take(unit));
}
API int fdsp_net_connect(fdsp_node* net, int s, int sp, int d, int dp) { return (net && net_connect(net->n, s, sp, d, dp)) ? FDSP_OK : fail(FDSP_ERR_ARG, "net_connect: bad port"); }
API int fdsp_net_connect_input(fdsp_node* net, int gi, int d, int dp) { return (net && net_connect_input(net->n, gi, d, dp)) ? FDSP_OK : fail(FDSP_ERR_ARG, "net_connect_input: bad port"); }
API int fdsp_net_connect_output(fdsp_node* net, int s, int sp, int go) { return (net && net_connect_output(net->n, s, sp, go)) ? FDSP_OK : fail(FDSP_ERR_ARG, "net_connect_output: bad port"); }
API int fdsp_net_pass_through(fdsp_node* net, int gi, int go) { return (net && net_pass_through(net->n, gi, go)) ? FDSP_OK : fail(FDSP_ERR_ARG, "net_pass_through: bad port"); }
API int fdsp_net_size(const fdsp_node* net) { return net ? net_size(net->n) : -1; }

API int fdsp_node_phase(fdsp_node* h, float phase) {  // src/combinator.rs:263-268
  if (!h) return fail(FDSP_ERR_ARG, "null node");
  Setting s; s.kind = P_PHASE; s.v[0] = phase; s.address.push_back({1, 1});
  h->n->set(s); h->n->reset();
  return FDSP_OK;
}
API int fdsp_node_seed(fdsp_node* h, uint64_t seed) {  // src/combinator.rs:270-276
  if (!h) return fail(FDSP_ERR_ARG, "null node");
  Setting s; s.kind = P_SEED; s.seed = seed; s.address.push_back({1, 0});
  h->n->set(s); h->n->reset();
  return FDSP_OK;
}
API int fdsp_node_set(fdsp_node* h, int kind, const float* v, int nv, uint64_t seed, const int64_t* addr, int naddr) {
  if (!h || nv < 0 || nv > 5 || naddr < 0 || naddr > 6 || (nv > 0 && !v) || (naddr > 0 && !addr)) return fail(FDSP_ERR_ARG, "bad setting");
  Setting s; s.kind = kind; s.seed = seed;
  for (int i = 0; i < nv; i++) s.v[i] = v[i];
  for (int i = 0; i < naddr; i++) s.address.push_back({(int)addr[2 * i], (uint64_t)addr[2 * i + 1]});
  h->n->set(s);
  return FDSP_OK;
}
API int fdsp_node_inputs(const fdsp_node* h) { return h ? h->n->inputs() : -1; }
API int fdsp_node_outputs(const fdsp_node* h) { return h ? h->n->outputs() : -1; }
API int fdsp_node_set_sample_rate(fdsp_node* h, double sr) { if (!h || !(sr > 0.0)) return fail(FDSP_ERR_ARG, "bad sample rate"); h->n->set_sample_rate(sr); return FDSP_OK; }
API uint64_t fdsp_node_id(const fdsp_node* h) { return h ? h->n->id() : 0; }
API uint64_t fdsp_node_ping(fdsp_node* h, int probe, uint64_t hash) { return h ? h->n->ping(probe != 0, AttoHash(hash)).state : 0; }
API int fdsp_node_leaf_hashes(fdsp_node* h, uint64_t* out, int max) {
  if (!h) return -1;
  std::vector<uint64_t> t;
  HNode::ping_trace() = &t;
  AttoHash a = h->n->ping(true, AttoHash(h->n->id()));
  h->n->ping(false, a);
  HNode::ping_trace() = nullptr;
  for (int i = 0; i < (int)t.size() && i < max; i++) out[i] = t[i];
  return (int)t.size();
}
API int fdsp_node_signature(const fdsp_node* h, char* out, int max) {
  if (!h || !out || max < 1) return -1;
  std::string s; h->n->sig(s);
  strncpy(out, s.c_str(), (size_t)max - 1); out[max - 1] = 0;
  return (int)s.size();
}
API int fdsp_node_lowering(const fdsp_node* h, uint32_t* P, int maxp, uint32_t* S, int maxs, uint32_t* U, int maxu, int* np, int* ns, int* nu) {
  if (!h || !np || !ns || !nu) return fail(FDSP_ERR_ARG, "node_lowering: bad arguments");
  Lowering l;
  h->n->lower(l);
  if (!l.ok) return fail(FDSP_ERR_UNSUPPORTED, l.why);
  *np = (int)l.P.size(); *ns = (int)l.S.size(); *nu = (int)l.U.size();
  for (int i = 0; i < *np && i < maxp && P; i++) P[i] = l.P[i];
  for (int i = 0; i < *ns && i < maxs && S; i++) S[i] = l.S[i];
  for (int i = 0; i < *nu && i < maxu && U; i++) U[i] = l.U[i];
  return FDSP_OK;
}
API int64_t fdsp_node_delay_floats(const fdsp_node* h) {   // floats of delay-line / ring storage the program of this node needs per voice
  if (!h) return -1;
  Lowering l;
  h->n->lower(l);
  if (!l.ok) return -1;
  int64_t t = 0;
  for (uint32_t d : l.dlen) t += d;
  return t;
}
API fdsp_node* fdsp_node_clone(const fdsp_node* h) { return h ? new (std::nothrow) fdsp_node{h->n->clone()} : nullptr; }
API void fdsp_node_free(fdsp_node* h) { if (h) { delete h->n; delete h; } }

API int fdsp_wavetable_count(int table) { return (table < 0 || table > 5) ? -1 : (int)global_wavetable(table).pitch.size(); }
API int fdsp_wavetable_info(int table, int index, float* pitch, int* length) {
  if (table < 0 || table > 5) return fail(FDSP_ERR_ARG, "bad table");
  const WaveTableHost& t = global_wavetable(table);
  if (index < 0 || index >= (int)t.pitch.size()) return fail(FDSP_ERR_ARG, "bad index");
  if (pitch) *pitch = t.pitch[index];
  if (length) *length = t.len[index];
  return FDSP_OK;
}
API const float* fdsp_wavetable_data(int table, int index) {
  if (table < 0 || table > 5) return nullptr;
  const WaveTableHost& t = global_wavetable(table);
  if (index < 0 || index >= (int)t.pitch.size()) return nullptr;
  return t.data.data() + t.off[index];
}

API int fdsp_bank_create(fdsp_node* const* voices, uint32_t nvoices, int device, uint32_t out_mode, fdsp_bank** out) {
  if (!voices || !out || nvoices == 0) return fail(FDSP_ERR_ARG, "bank_create: bad arguments");
  std::vector<HNode*> v;
  bool null_voice = false;
  for (uint32_t i = 0; i < nvoices; i++) { if (!voices[i]) null_voice = true; v.push_back(take(voices[i])); }
  if (null_voice) { for (HNode* n : v) delete n; return fail(FDSP_ERR_ARG, "bank_create: null voice"); }
  fdsp_bank* b = new (std::nothrow) fdsp_bank();
  if (!b) { for (HNode* n : v) delete n; return fail(FDSP_ERR_ARG, "out of memory"); }
  std::string e = b->b.init(v, device, out_mode);
  if (!e.empty()) { for (HNode* n : v) delete n; delete b; return status(e); }
  *out = b;
  return FDSP_OK;
}
API int fdsp_bank_create_from_net(fdsp_node* net, int device, uint32_t out_mode, fdsp_bank** out) {
  if (!net || !out) return fail(FDSP_ERR_ARG, "bank_create_from_net: bad arguments");
  std::vector<HNode*> v; std::string tree, err; std::vector<int> ids;
  HNode* n = take(net);
  const bool ok = net_extract_voices(n, v, tree, err, &ids);
  delete n;
  if (!ok) { for (HNode* x : v) delete x; return fail(FDSP_ERR_UNSUPPORTED, "no device lowering for this Net: " + err); }
  fdsp_bank* b = new (std::nothrow) fdsp_bank();
  if (!b) { for (HNode* x : v) delete x; return fail(FDSP_ERR_STATE, "out of memory"); }
  b->b.tree_mix = tree == "pairwise" ? 1 : 2; b->b.net_rate = true; b->b.vertex_of_voice = ids;
  std::string e = b->b.init(v, device, out_mode);
  if (!e.empty()) { for (HNode* x : v) delete x; delete b; return status(e); }
  *out = b;
  return FDSP_OK;
}
API int fdsp_bank_voice_of_vertex(const fdsp_bank* b, int vertex) {
  if (!b) return -1;
  for (size_t i = 0; i < b->b.vertex_of_voice.size(); i++) if (b->b.vertex_of_voice[i] == vertex) return (int)i;
  return -1;
}
API void fdsp_bank_destroy(fdsp_bank* b) { delete b; }
API int fdsp_bank_clone(const fdsp_bank* b, fdsp_bank** out) {
  if (!b || !out) return fail(FDSP_ERR_ARG, "null bank");
  fdsp_bank* c = new (std::nothrow) fdsp_bank();
  if (!c) return fail(FDSP_ERR_STATE, "out of memory");
  std::string e = b->b.clone_into(c->b);
  if (!e.empty()) { delete c; return status(e); }
  *out = c;
  return FDSP_OK;
}
API uint32_t fdsp_bank_voices(const fdsp_bank* b) { return b ? b->b.V() : 0; }
API int fdsp_bank_inputs(const fdsp_bank* b) { return b ? b->b.nin : -1; }
API int fdsp_bank_voice_outputs(const fdsp_bank* b) { return b ? b->b.nout : -1; }
API int fdsp_bank_outputs(const fdsp_bank* b) { return !b ? -1 : ((b->b.out_mode & 2u) ? b->b.nout : (int)(b->b.V() * (uint32_t)b->b.nout)); }
API int fdsp_bank_set_sample_rate(fdsp_bank* b, double sr) { return b ? status(b->b.set_sample_rate(sr)) : fail(FDSP_ERR_ARG, "null bank"); }
API int fdsp_bank_set(fdsp_bank* b, uint32_t voice, int kind, const float* v, int nv, uint64_t seed, const int64_t* addr, int naddr) {
  if (!b || nv < 0 || nv > 5 || naddr < 0 || naddr > 6 || (nv > 0 && !v) || (naddr > 0 && !addr)) return fail(FDSP_ERR_ARG, "bad setting");
  Setting s; s.kind = kind; s.seed = seed;
  for (int i = 0; i < nv; i++) s.v[i] = v[i];
  for (int i = 0; i < naddr; i++) s.address.push_back({(int)addr[2 * i], (uint64_t)addr[2 * i + 1]});
  std::string e = b->b.set(voice, s);
  return status(e, FDSP_ERR_ARG);
}
// ---- JIT cache (csrc/host/jit.cpp): compiled units are kept on disk next to the library; a machine without a GPU can fill it
API int fdsp_jit_precompile(const char* signature, int mode, int table_variant) {
  if (!signature) return fail(FDSP_ERR_ARG, "null signature");
  if (find_kernel(signature)) return FDSP_OK;   // ahead-of-time class: nothing to compile
  std::string e = jit_precompile(signature, mode, table_variant & 1, table_variant >> 8);   // bits 8..: width (32 / 128) of the stage-pipelined kernel, 0 = plain
  return e.empty() ? FDSP_OK : fail(FDSP_ERR_UNSUPPORTED, e);
}
API void fdsp_jit_cache_stats(int* hits, int* nvrtc_runs) { jit_cache_stats(hits, nvrtc_runs); }
// ---- WAV edge (src/write.rs): planar f32 [channels][stride] -> the reference's file bytes, and back
API int fdsp_wave_save(const char* path, const float* planar, uint32_t channels, uint64_t length, uint64_t stride, double sample_rate, int bits) {
  std::string e = wav_write(path, planar, channels, length, stride, sample_rate, bits);
  return e.empty() ? FDSP_OK : fail(FDSP_ERR_ARG, e);
}
API int64_t fdsp_wave_encode(uint8_t* out, uint64_t max, const float* planar, uint32_t channels, uint64_t length, uint64_t stride, double sample_rate, int bits) {
  std::vector<uint8_t> b;
  std::string e = wav_encode(b, planar, channels, length, stride, sample_rate, bits);
  if (!e.empty()) { fail(FDSP_ERR_ARG, e); return -1; }
  if (out && max >= b.size()) memcpy(out, b.data(), b.size());
  return (int64_t)b.size();
}
API int fdsp_wave_load(const char* path, float* planar, uint64_t max_floats, uint32_t* channels, uint64_t* length, double* sample_rate) {
  if (!channels || !length || !sample_rate) return fail(FDSP_ERR_ARG, "wave_load: null output");
  std::vector<float> p;
  std::string e = wav_read(path, p, channels, length, sample_rate);
  if (!e.empty()) return fail(FDSP_ERR_ARG, e);
  if (planar && max_floats >= p.size()) memcpy(planar, p.data(), p.size() * 4);   // call once with planar = NULL to size the buffer
  return FDSP_OK;
}
// ---- sequencer banks: voices made by fdsp_event
API int fdsp_bank_edit_event(fdsp_bank* b, uint32_t voice, double end_time, double fade_out) {
  if (!b) return fail(FDSP_ERR_ARG, "null bank");
  std::string e = b->b.edit_event(voice, end_time, fade_out);
  return status(e, FDSP_ERR_ARG);
}
API int fdsp_bank_replace_voice(fdsp_bank* b, uint32_t voice, fdsp_node* unit) {
  if (!b) { fdsp_node_free(unit); return fail(FDSP_ERR_ARG, "null bank"); }
  std::string e = b->b.replace_voice(voice, take(unit));
  return status(e, FDSP_ERR_ARG);
}
API int fdsp_bank_crossfade_voice(fdsp_bank* b, uint32_t voice, int fade_ease, float fade_time, fdsp_node* unit) {
  if (!b) { fdsp_node_free(unit); return fail(FDSP_ERR_ARG, "null bank"); }
  std::string e = b->b.crossfade_voice(voice, fade_ease, fade_time, take(unit));
  return status(e, FDSP_ERR_ARG);
}
API int fdsp_bank_remove_voice(fdsp_bank* b, uint32_t voice) {
  if (!b) return fail(FDSP_ERR_ARG, "null bank");
  std::string e = b->b.remove_voice(voice);
  return status(e, FDSP_ERR_ARG);
}
API int fdsp_bank_push_event(fdsp_bank* b, fdsp_node* event, uint32_t* voice) {
  if (!b || !event) { fdsp_node_free(event); return fail(FDSP_ERR_ARG, "null bank or event"); }
  HNode* keep = event->n->clone();                   // push_event consumes its node; the slow path needs it again
  std::string e = b->b.push_event(take(event), voice);
  if (e.empty()) { delete keep; return FDSP_OK; }
  if (tag_of(e) != 'N') { delete keep; return status(e, FDSP_ERR_ARG); }   // anything but "no finished event of this class is free"
  e = b->b.add_voice(keep, voice);                   // no free slot of this class: grow the bank (running state of the others preserved)
  return status(e, FDSP_ERR_ARG);
}
API int fdsp_bank_add_voice(fdsp_bank* b, fdsp_node* unit, uint32_t* voice) {
  if (!b || !unit) { fdsp_node_free(unit); return fail(FDSP_ERR_ARG, "null bank or unit"); }
  std::string e = b->b.add_voice(take(unit), voice);
  return status(e, FDSP_ERR_ARG);
}
API int fdsp_bank_slot_set(fdsp_bank* b, uint32_t voice, int fade_ease, double fade_time, fdsp_node* unit) {
  if (!b) { fdsp_node_free(unit); return fail(FDSP_ERR_ARG, "null bank"); }
  std::string e = b->b.slot_set(voice, fade_ease, fade_time, take(unit));
  return status(e, FDSP_ERR_ARG);
}
API double fdsp_bank_time(const fdsp_bank* b) { return b ? b->b.seq_time : 0.0; }
API int fdsp_bank_reset(fdsp_bank* b) { return b ? status(b->b.reset()) : fail(FDSP_ERR_ARG, "null bank"); }
API int fdsp_bank_allocate(fdsp_bank* b, uint64_t max_n) {
  if (!b) return fail(FDSP_ERR_ARG, "null bank");
  uint32_t chunk = (uint32_t)std::min<uint64_t>(16384, std::max<uint64_t>(64, (max_n + 63) / 64 * 64));
  return status(b->b.ensure_staging(chunk));
}
API int fdsp_bank_process(fdsp_bank* b, uint32_t size, const float* in, float* out) {
  if (!b || !out) return fail(FDSP_ERR_ARG, "null bank or output");
  return status(b->b.process(size, in, out));
}
API int fdsp_bank_render(fdsp_bank* b, uint64_t n, const float* in, float* out_voices, float* out_mix) {
  if (!b) return fail(FDSP_ERR_ARG, "null bank");
  return status(b->b.render_host(n, in, out_voices, out_mix));
}
API int fdsp_bank_render_device(fdsp_bank* b, uint64_t n, const float* in_dev, uint64_t in_stride, float* out_dev, uint64_t out_stride,
                                float* mix_dev, uint64_t mix_stride) {
  if (!b) return fail(FDSP_ERR_ARG, "null bank");
  return status(b->b.render_device(n, in_dev, in_stride, out_dev, out_stride, mix_dev, mix_stride));
}
// ---- multi-GPU mix-down (host/group.h)
struct fdsp_group { fdsp::host::Group* g; };
API int fdsp_group_unique_id(void* id, uint64_t bytes) {
  if (!id || bytes < 128) return fail(FDSP_ERR_ARG, "the id buffer must hold 128 bytes");
  return status(fdsp::host::group_unique_id(id));
}
API int fdsp_group_create(int nranks, int rank, const void* id, int device, fdsp_group** out) {
  if (!out) return fail(FDSP_ERR_ARG, "null out pointer");
  fdsp::host::Group* g = nullptr;
  std::string e = fdsp::host::group_create(nranks, rank, id, device, &g);
  if (!e.empty()) return status(e);
  fdsp_group* h = new (std::nothrow) fdsp_group();
  if (!h) { delete g; return fail(FDSP_ERR_STATE, "out of memory"); }
  h->g = g; *out = h;
  return FDSP_OK;
}
API void fdsp_group_destroy(fdsp_group* g) { if (g) { delete g->g; delete g; } }
API int fdsp_group_rank(const fdsp_group* g) { return g ? g->g->rank : -1; }
API int fdsp_group_size(const fdsp_group* g) { return g ? g->g->nranks : -1; }
API int fdsp_bank_render_reduced(fdsp_bank* b, fdsp_group* g, uint64_t n, const float* in, float* out_mix, int root) {
  if (!b || !g) return fail(FDSP_ERR_ARG, "null bank or group");
  return status(fdsp::host::group_render_host(b->b, *g->g, n, in, out_mix, root));
}
API int fdsp_bank_reduce_device(fdsp_bank* b, fdsp_group* g, uint64_t n, float* mix_dev, uint64_t mix_stride, int root) {
  if (!b || !g) return fail(FDSP_ERR_ARG, "null bank or group");
  return status(fdsp::host::group_reduce_device(b->b, *g->g, n, mix_dev, mix_stride, root));
}
API int fdsp_bank_sync(fdsp_bank* b) {
  if (!b) return fail(FDSP_ERR_ARG, "null bank");
  cudaSetDevice(b->b.device);
  { std::string re = b->b.rt_stop(); if (!re.empty()) return status(re); }
  cudaError_t e = cudaStreamSynchronize(b->b.stream);
  if (e != cudaSuccess) return fail(FDSP_ERR_CUDA, cudaGetErrorString(e));
  if (cudaEventElapsedTime(&b->b.last_ms, b->b.ev0, b->b.ev1) != cudaSuccess) b->b.last_ms = 0.0f;
  // time covered by the voice kernels: the union of their [begin, end] intervals measured from ev0 (classes of a multi-class bank run on
  // concurrent streams, so a plain sum of the durations would exceed the step)
  b->b.last_dom_ms = 0.0f;
  std::vector<std::pair<float, float>> iv;
  for (size_t i = 0; i + 1 < b->b.dom_n; i += 2) {
    float t0 = 0.0f, t1 = 0.0f;
    if (cudaEventElapsedTime(&t0, b->b.ev0, b->b.dom_ev[i]) == cudaSuccess && cudaEventElapsedTime(&t1, b->b.ev0, b->b.dom_ev[i + 1]) == cudaSuccess && t1 > t0)
      iv.emplace_back(t0, t1);
  }
  std::sort(iv.begin(), iv.end());
  float hi = -1.0f;
  for (auto& q : iv) { if (q.second <= hi) continue; b->b.last_dom_ms += q.second - std::max(q.first, hi); hi = q.second; }
  return FDSP_OK;
}
API void* fdsp_bank_stream(fdsp_bank* b) { return b ? (void*)b->b.stream : nullptr; }
API int fdsp_bank_num_classes(const fdsp_bank* b) { return b ? (int)b->b.classes.size() : -1; }
API int fdsp_bank_class_info(const fdsp_bank* b, int cls, char* sig, int max, uint32_t* voices, uint32_t* state_words, uint32_t* param_words,
                             uint64_t* delay_floats) {
  if (!b || cls < 0 || cls >= (int)b->b.classes.size()) return fail(FDSP_ERR_ARG, "bad class index");
  const VoiceClass& c = b->b.classes[cls];
  if (sig && max > 0) { strncpy(sig, c.sig.c_str(), (size_t)max - 1); sig[max - 1] = 0; }
  if (voices) *voices = c.V();
  if (state_words) *state_words = c.ns;
  if (param_words) *param_words = c.np;
  if (delay_floats) *delay_floats = c.dl_floats + c.ring_floats;
  return FDSP_OK;
}
API int fdsp_bank_class_stages(const fdsp_bank* b, int cls) {
  if (!b || cls < 0 || cls >= (int)b->b.classes.size()) return -1;
  const VoiceClass& c = b->b.classes[cls];
  return c.k ? c.k->stages : 1;
}
API uint64_t fdsp_bank_launch_count(const fdsp_bank* b) { return b ? b->b.launches : 0; }
API float fdsp_bank_last_kernel_ms(const fdsp_bank* b) { return b ? b->b.last_ms : 0.0f; }
API float fdsp_bank_last_dominant_ms(const fdsp_bank* b) { return b ? b->b.last_dom_ms : 0.0f; }

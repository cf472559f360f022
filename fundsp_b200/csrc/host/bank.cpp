// fundsp_b200 bank runtime implementation — see bank.h.
#include "bank.h"
#include "../dsp/fdn_args.h"

#include <algorithm>
#include <mutex>
#include <cmath>
#include <limits>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>

namespace fdsp {
namespace host {

namespace {
constexpr uint32_t TIME_CHUNK = 16384;  // samples per launch (multiple of 64): bounds the partial-mix buffer
// sub-chunk of two-stage (dry program -> FDN reverb) classes: stage 1 of chunk k+1 overlaps stage 2 of chunk k
constexpr uint32_t PIPE_CHUNK = 2048;

// the runtime's own calls (which return "" or the message) inside a function of the same convention
#define TRY(call) do { std::string e_ = (call); if (!e_.empty()) return e_; } while (0)

// the class (or the saved state of one, regroup) whose ascending `voices` hold `voice`, and the voice's column there; nullptr: none
template <class C> C* locate(std::vector<C>& classes, uint32_t voice, uint32_t* col) {
  for (auto& c : classes) {
    auto it = std::lower_bound(c.voices.begin(), c.voices.end(), voice);
    if (it != c.voices.end() && *it == voice) { *col = (uint32_t)(it - c.voices.begin()); return &c; }
  }
  return nullptr;
}
}  // namespace
static_assert(!std::is_copy_constructible<VoiceClass>::value, "a copy of a class would free its buffers twice");

// `sig` is `Pipe<X,tail>`: *front = X
static bool pipe_into(const std::string& sig, const std::string& tail, std::string* front) {
  const std::string t = "," + tail + ">";
  if (sig.size() <= 5 + t.size() || sig.compare(0, 5, "Pipe<") != 0 || sig.compare(sig.size() - t.size(), t.size(), t) != 0) return false;
  *front = sig.substr(5, sig.size() - 5 - t.size());
  return true;
}

// The form of class c (see Form), from the lowering `l` of one of its voices, and the signature of its program (empty: an FDN class
// without a dry stage). `wet`: the FDN tail adds the reverb to the dry signal on a stereo bus.
static Form choose_form(const VoiceClass& c, const Lowering& l, int nin, int nout, bool one_class, std::string* prog, bool* wet) {
  static const std::string REV = "Pipe<Pipe<MultiSplit<2,16>,Feedback<1,Multi<30,0,32,Pipe<Delay,Fir<3>>>>>,Binop<2,Multi<31,0,32,Panner<1>>,Constant<2>>>";
  static const std::string BUS = "Bus<MultiPass<2>,Unop<3," + REV + ">>";   // dry + g * reverb on a stereo bus
  *prog = c.sig; *wet = false;
  if (!getenv("FDSP_DISABLE_FDN")) {   // A/B switch: run reverbs in the generic thread-per-voice form
    std::string front;
    bool fdn = true;
    if ((c.sig == REV || c.sig == BUS) && nin == 2) *wet = c.sig == BUS;
    else if (pipe_into(c.sig, BUS, &front)) *wet = true;
    else if (!pipe_into(c.sig, REV, &front)) fdn = false;
    // the kernel's prefetch distance needs every delay >= 192 samples
    for (size_t k = c.nu - 32; fdn && k < c.nu; k++) fdn = c.uniform[k] >= FDN_MIN_RING;
    if (fdn) { *prog = front; return Form::fdn; }
    *wet = false;
  }
#ifndef FDSP_HOST_EMUL   // (not on the CPU mock device)
  // `X >> convolve(h)` with a response long enough for 128-wide tiles goes to tensor cores (FDSP_TC_CONV=0: direct form only; FDSP_TC_MINK:
  // shortest response, default 32 taps). One output channel, and one class: its mix-down is the voice-order fold of its own rows.
  const char* e = getenv("FDSP_TC_CONV"); const char* m = getenv("FDSP_TC_MINK");
  std::string front;
  if (one_class && nout == 1 && !(e && atoi(e) == 0) && pipe_into(c.sig, "Convolver", &front) && l.conv_K >= (m ? (uint32_t)atoi(m) : 32u) &&
      l.conv_off + 2u + l.conv_K == c.nu) {
    *prog = front;
    return Form::conv;
  }
#endif
  return Form::plain;
}

// Per form: the words of a class's lowering that its tail holds rather than its program (FDN: the reverb's, plus the gain of a wet bus;
// conv: the Convolver's state word, its ring index, and two uniform words, which stay in the class's layout unused like its history
// ring), the program's output channels (0: the bank's), and the wording of the errors about the program.
struct FormRule { uint32_t tail_p, tail_s, tail_u; int out; const char *name, *name_end, *layout, *layout_end; };
static const FormRule FORM_RULES[] = {
    /* plain */ {0, 0, 0, 0, "graph class `", "`", "host lowering of `", "` disagrees with the device word layout"},
    /* fdn */ {162, 160, 32, 2, "the dry stage `", "`", "dry-stage layout of `", "` disagrees with the host lowering"},
    /* conv */ {0, 1, 2, 1, "`", "` (in front of the convolver)", "layout of `", "` in front of the convolver disagrees with the host lowering"},
};

namespace {
std::mutex g_rt_mu;          // registry of the bank that owns each device's resident process() kernel (see rt_stop)
Bank* g_rt_owner[64] = {};
}
Bank::~Bank() {
  cudaSetDevice(device);
  rt_stop();
  if (device >= 0 && device < 64) { std::lock_guard<std::mutex> lock(g_rt_mu); if (g_rt_owner[device] == this) g_rt_owner[device] = nullptr; }
}

std::string Bank::init(std::vector<HNode*>& voices, int dev, uint32_t mode) {
  device = dev; out_mode = mode;
  for (HNode* v : voices) nodes.emplace_back(v);
  voices.clear();
  if (nodes.empty()) return "#A bank needs at least one voice";
  if ((mode & 3u) == 0u) return "#A out_mode must include FDSP_OUT_VOICES and/or FDSP_OUT_MIX";
  nin = nodes[0]->inputs(); nout = nodes[0]->outputs();
  if (nout < 1) return "#A voices must have at least one output";
  for (auto& n : nodes) if (n->inputs() != nin || n->outputs() != nout) return "#A all voices of a bank must agree on inputs() and outputs()";
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= dev) return "no usable CUDA device: fundsp_b200 has no CPU fallback";
  CU(cudaSetDevice(device));
  TRY(rt_stop());   // (another bank's resident process() kernel would make the allocations below wait for its idle time-out)
  // `stream` carries the latency-bound voice programs (few CTAs, long serial chains) and gets the highest priority, so that in
  // the two-stage pipeline its CTAs are placed before the wide FDN kernel of the previous chunk (stream2) fills every SM.
  int prio_lo = 0, prio_hi = 0;
  CU(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
  CU(cudaStreamCreateWithPriority(stream.put(), cudaStreamNonBlocking, prio_hi));
  CU(cudaStreamCreateWithPriority(stream2.put(), cudaStreamNonBlocking, prio_lo));
  CU(cudaEventCreate(ev0.put())); CU(cudaEventCreate(ev1.put())); CU(cudaEventCreateWithFlags(e_begin.put(), cudaEventDisableTiming));
  TRY(d_ticket.grow(1)); CU(cudaMemsetAsync(d_ticket, 0, 4, stream));
  return lower_and_upload(true);
}

// the FDN rings and the convolver's history columns (with the rows behind them)
std::string VoiceClass::clear_history(cudaStream_t st) {
  if (ring_floats) CU(cudaMemsetAsync(d_ring, 0, (size_t)ring_floats * V() * sizeof(float), st));
  if (form == Form::conv) {
    CU(cudaMemsetAsync(d_cx, 0, (size_t)V() * conv_stride * sizeof(float), st));
    CU(cudaMemsetAsync(d_cxl, 0, (size_t)V() * conv_stride * sizeof(float), st));
  }
  return "";
}

std::string Bank::lower_and_upload(bool upload_state) {
  CU(cudaSetDevice(device));
  TRY(rt_end_streak());
  // a looping sequencer (ReplayMode::Loop): every event of the bank carries the sequencer's loop period
  {
    double la = 0.0; bool any = false; size_t events = 0;
    for (auto& n : nodes) { double t = 0.0; if (!event_loop(n.get(), &t)) continue; events++; if (!any) { la = t; any = true; } else if (t != la) return "#U the events of one bank belong to one sequencer: their loop periods differ"; }
    if (la > 0.0 && events != nodes.size()) return "#U a looping sequencer bank holds events only";
    loop_arg = la;
  }
  // 1. lower every voice, group into classes keyed by (type expression, uniform words)
  struct Low { std::string key; Lowering l; std::string sig; };
  std::vector<Low> lows(nodes.size());
  std::map<std::string, int> index;
  std::vector<VoiceClass> fresh;
  for (size_t v = 0; v < nodes.size(); v++) {
    Low& lo = lows[v];
    nodes[v]->sig(lo.sig);
    nodes[v]->lower(lo.l);
    if (!lo.l.ok) return "#U voice " + std::to_string(v) + ": " + lo.l.why;
    lo.key = lo.sig + "|";
    lo.key.append((const char*)lo.l.U.data(), lo.l.U.size() * 4);
    auto it = index.find(lo.key);
    int ci;
    if (it == index.end()) {
      ci = (int)fresh.size(); index[lo.key] = ci;
      VoiceClass c; c.sig = lo.sig; c.uniform = lo.l.U;
      c.np = (uint32_t)lo.l.P.size(); c.ns = (uint32_t)lo.l.S.size(); c.nu = (uint32_t)lo.l.U.size();
      fresh.push_back(std::move(c));
    } else ci = it->second;
    fresh[ci].voices.push_back((uint32_t)v);
    std::string().swap(lo.key); std::vector<uint32_t>().swap(lo.l.U);   // the class keeps the uniform words (a sampler voice's may be a whole wave)
  }
  // then the form of each class, its program and the layout that program must have (the class's first voice gives its layout)
  for (auto& c : fresh) {
    const Lowering& l = lows[c.voices[0]].l;
    std::string prog; bool wet = false;
    c.form = choose_form(c, l, nin, nout, fresh.size() == 1, &prog, &wet);
    const size_t nd_lines = c.form == Form::fdn ? l.dlen.size() - 32 : l.dlen.size();   // the last 32 lines of an FDN class live in its rings
    for (size_t k = 0; k < l.dlen.size(); k++) { if (k < nd_lines) c.dl_floats += l.dlen[k]; else c.ring_floats += fdn_ring_phys(l.dlen[k]); }
    if (c.form == Form::fdn) {
      c.p0 = c.np - 162; c.s0 = c.ns - 160; c.u0 = c.nu - 32;
      c.scalar_row = wet ? (int)c.p0 - 1 : -1;
    } else if (c.form == Form::conv) {
      c.conv_K = l.conv_K; c.conv_off = l.conv_off;
      c.conv_H = (c.conv_K - 1u + 31u) / 32u * 32u; if (c.conv_H == 0) c.conv_H = 32;
      c.conv_J = conv_tc_toeplitz_cols(c.conv_K); c.conv_stride = c.conv_H + TIME_CHUNK;
    }
    if (!prog.empty()) {
      const FormRule& r = FORM_RULES[(int)c.form];
      std::string jerr;
      c.k = get_program(prog, device, jerr);
      if (!c.k) return std::string("#U no device program for ") + r.name + prog + r.name_end + ": " + jerr;
      // extraP / extraU: variable-length data behind the words the device templates count
      if ((uint32_t)c.k->NP != c.np - l.extraP - r.tail_p - (wet ? 1u : 0u) || (uint32_t)c.k->NS != c.ns - r.tail_s ||
          (uint32_t)c.k->NU != c.nu - l.extraU - r.tail_u || c.k->IN != nin || c.k->OUT != (r.out ? r.out : nout))
        return std::string("internal: ") + r.layout + prog + r.layout_end;
    }
    // reset exemptions of this graph class, in the class's own word / delay-line coordinates
    for (auto& q : l.keepS) if (q.second > q.first) c.keep_s.emplace_back(q.first, q.second);
    std::vector<uint64_t> doff(l.dlen.size() + 1, 0);
    for (size_t k = 0; k < l.dlen.size(); k++) doff[k + 1] = doff[k] + (k < nd_lines ? l.dlen[k] : 0u);
    for (auto& q : l.keepD) if (q.second > q.first && q.second <= nd_lines) c.keep_d.emplace_back(doff[q.first], doff[q.second]);
    std::sort(c.keep_s.begin(), c.keep_s.end()); std::sort(c.keep_d.begin(), c.keep_d.end());
  }
  sh_uses.assign(nodes.size(), {});
  for (size_t v = 0; v < nodes.size(); v++) sh_uses[v] = lows[v].l.shared;
  TRY(sh_check(0, sh_uses[0]));
  // 2. keep device buffers of classes that survive unchanged (same key order / sizes), else rebuild
  const bool same_shape = classes.size() == fresh.size() && std::equal(classes.begin(), classes.end(), fresh.begin(), [](const VoiceClass& a, const VoiceClass& b) {
                            return a.sig == b.sig && a.voices == b.voices && a.uniform == b.uniform; });
  if (!same_shape) {
    classes = std::move(fresh);   // (releases the old classes' buffers)
    upload_state = true;
  }
  for (auto& c : classes) {
    const uint32_t V = c.V(); const int NP = (int)c.np, NS = (int)c.ns;
    std::vector<uint32_t> P((size_t)NP * V), S((size_t)NS * V), rows(V), id;
    for (uint32_t i = 0; i < V; i++) {
      const Lowering& l = lows[c.voices[i]].l;
      for (int k = 0; k < NP; k++) P[(size_t)k * V + i] = l.P[k];
      for (int k = 0; k < NS; k++) S[(size_t)k * V + i] = l.S[k];
      rows[i] = c.voices[i] * (uint32_t)nout;
    }
    c.state0 = S; c.state0_stale = true;
    for (uint32_t i = 0; i < V; i++)   // the words whose reset value differs from their starting value (Lowering::resetS)
      for (auto& w : lows[c.voices[i]].l.resetS) if (w.first < (uint32_t)NS) c.state0[(size_t)w.first * V + i] = w.second;
    if (!same_shape) {
      TRY(c.d_params.grow(P.size()));
      TRY(c.d_state.grow(S.size()));
      TRY(c.d_uniform.grow(c.uniform.size()));
      TRY(c.d_rowmap.grow(rows.size()));
      TRY(c.d_dline.grow((size_t)c.dl_floats * V));
      if (c.form == Form::fdn) TRY(c.d_ring.grow((size_t)c.ring_floats * V));
      if (c.fdn_with_dry()) {
        TRY(c.d_dry.grow((size_t)V * 2 * TIME_CHUNK));
        TRY(c.d_dry2.grow((size_t)V * 2 * PIPE_CHUNK));
        for (int q = 0; q < 2; q++) { CU(cudaEventCreateWithFlags(c.e_dry[q].put(), cudaEventDisableTiming)); CU(cudaEventCreateWithFlags(c.e_fdn[q].put(), cudaEventDisableTiming)); }
      }
      if (c.form == Form::conv) {
        TRY(c.d_cx.grow((size_t)V * c.conv_stride));
        TRY(c.d_cxl.grow((size_t)V * c.conv_stride));
        TRY(c.d_th.grow((size_t)128 * c.conv_J));
        TRY(c.d_tl.grow((size_t)128 * c.conv_J));
        CU(conv_tc_make_maps(c.d_cx, c.d_cxl, V, c.conv_stride, c.d_th, c.d_tl, c.conv_J, &c.conv_maps));
      }
      if (c.fdn_with_dry() || c.form == Form::conv) {   // the rows the dry stage writes (two per voice) or the convolver reads (one per voice)
        TRY(c.d_dryrows.grow(V));
        id.resize(V);
        for (uint32_t i = 0; i < V; i++) id[i] = c.form == Form::conv ? i : 2 * i;
        CU(cudaMemcpyAsync(c.d_dryrows, id.data(), V * 4, cudaMemcpyHostToDevice, stream));
      }
      CU(cudaMemcpyAsync(c.d_rowmap, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, stream));
      if (!c.uniform.empty()) CU(cudaMemcpyAsync(c.d_uniform, c.uniform.data(), c.uniform.size() * 4, cudaMemcpyHostToDevice, stream));
    }
    if (!P.empty()) CU(cudaMemcpyAsync(c.d_params, P.data(), P.size() * 4, cudaMemcpyHostToDevice, stream));
    if (upload_state) {
      if (!S.empty()) CU(cudaMemcpyAsync(c.d_state, S.data(), S.size() * 4, cudaMemcpyHostToDevice, stream));
      if (c.dl_floats) CU(cudaMemsetAsync(c.d_dline, 0, (size_t)c.dl_floats * V * sizeof(float), stream));
      TRY(c.clear_history(stream));
      if (c.form == Form::conv) CU(launch_conv_toeplitz(reinterpret_cast<const float*>(c.d_uniform + c.conv_off + 2), c.conv_K, c.d_th, c.d_tl, c.conv_J, stream));
    }
    CU(cudaStreamSynchronize(stream));   // P, S, rows and id are pageable and go out of scope
  }
  // 3. wavetables used by any class (a class that arrives later — add_voice — may bring a waveform the bank has not loaded yet)
  {
    bool changed = false;
    for (int kind = 0; kind < 6; kind++) {
      if (d_wtdata[kind]) continue;
      bool used = false;
      const std::string tag = "WaveSynth<" + std::to_string(kind) + ",", tag2 = "PhaseSynth<" + std::to_string(kind) + ">";
      for (auto& c : classes) used = used || c.sig.find(tag) != std::string::npos || c.sig.find(tag2) != std::string::npos;
      if (!used) continue;
      const WaveTableHost& t = device_wavetable(kind);
      h_wt[kind].n = (int)t.pitch.size(); h_wt[kind].total = (int)t.data.size();
      for (size_t i = 0; i < t.pitch.size() && i < 48; i++) { h_wt[kind].pitch[i] = t.pitch[i]; h_wt[kind].off[i] = t.off[i]; h_wt[kind].len[i] = t.len[i]; }
      TRY(d_wtdata[kind].grow(t.data.size()));
      CU(cudaMemcpyAsync(d_wtdata[kind], t.data.data(), t.data.size() * 4, cudaMemcpyHostToDevice, stream));
      h_wt[kind].data = d_wtdata[kind];
      changed = true;
    }
    if (!d_wt) { TRY(d_wt.grow(6)); changed = true; }
    if (changed) { CU(cudaMemcpyAsync(d_wt, h_wt, sizeof(h_wt), cudaMemcpyHostToDevice, stream)); CU(cudaStreamSynchronize(stream)); }   // (h_wt is pageable)
  }
  if (upload_state) dirty = false;
  return sh_rebuild();
}

std::string Bank::set_sample_rate(double s) {  // AudioUnit::set_sample_rate
  sr = s;
  for (auto& n : nodes) {   // the bank of a sequencer is re-rated like the sequencer: its events' units are reset (a unit pushed later is not)
    const bool reset = event_rerate_resets(n.get(), unit_rate());
    n->set_sample_rate(unit_rate());
    if (reset) n->reset();
  }
  // Parameters always follow the new rate. State is re-initialised only while nothing has been rendered
  // (or when delay lengths change, which resets the lines like src/delay.rs:105-113).
  return lower_and_upload(!dirty);
}

std::string Bank::set(uint32_t voice, const Setting& st) {  // AudioUnit::set (src/audiounit.rs:62, src/setting.rs) on a live bank
  if (voice >= V()) return "#A set: voice index out of range";
  CU(cudaSetDevice(device));
  TRY(rt_end_streak());
  // the setting is tried on a COPY of the voice's host graph: a refused setting (one that would change a class-uniform word) leaves
  // both the host graph and the device untouched; the copy replaces the original only after the upload
  std::unique_ptr<HNode> trial(nodes[voice]->clone());
  trial->set(st);
  Lowering l;
  trial->lower(l);
  if (!l.ok) return "#U " + l.why;
  uint32_t i = 0;
  if (VoiceClass* cp = locate(classes, voice, &i)) {
    VoiceClass& c = *cp;
    const uint32_t Vc = c.V();
    if (l.U != c.uniform || l.P.size() != c.np || l.S.size() != c.ns)
      return "#U set: the setting changes a class-uniform word (a delay length); rebuild the bank instead";
    TRY(sh_check(voice, l.shared));
    // parameters take effect at once (one strided column of the [NP][V] block); running state is left alone, the
    // construction-time state (what reset() restores) follows the setting like the reference's stored phase/seed
    if (c.np) CU(cudaMemcpy2DAsync(c.d_params + i, (size_t)Vc * 4, l.P.data(), 4, 4, c.np, cudaMemcpyHostToDevice, stream));
    CU(cudaStreamSynchronize(stream));  // `l` is pageable and goes out of scope
    const std::vector<uint32_t> S0 = l.reset_image();
    for (uint32_t k = 0; k < c.ns; k++) c.state0[(size_t)k * Vc + i] = S0[k];
    c.state0_stale = true;
    nodes[voice] = std::move(trial);
    sh_uses[voice] = l.shared;
    return sh_rebuild();
  }
  return "internal: voice not found in any class";
}

double Bank::loop_point() const {
  if (!(loop_arg > 0.0)) return std::numeric_limits<double>::infinity();
  const double ur = unit_rate();
  return std::max(64.0 * (1.0 / ur), std::round(loop_arg * ur) / ur);
}
void Bank::advance_clock(uint64_t n) {   // what every Event<X> voice does to its own clock (nodes.cuh Event::plan / at_sample)
  const double ur = unit_rate(), sd = 1.0 / ur, lp = loop_point();
  for (uint64_t t0 = 0; t0 < n; t0 += 64) {
    const uint64_t size = std::min<uint64_t>(64, n - t0);
    if (!(loop_arg > 0.0)) { seq_time = seq_time + sd * (double)size; continue; }
    const double x = std::round(std::max(0.0, lp - seq_time) * ur);
    const uint64_t loop_size = x > 0.0 ? (uint64_t)x : 0;
    seq_time = std::min(seq_time + sd * (double)size, lp);
    if (loop_size < size) seq_time = std::min(0.0 + sd * (double)(size - loop_size), lp);   // wrapped: the rest of the block counts from 0
  }
}
std::string Bank::state0_to_device(VoiceClass& c, const uint32_t** out) {
  *out = nullptr;
  if (!(loop_arg > 0.0) || c.state0.empty() || c.sig.compare(0, 6, "Event<") != 0) return "";
  if (!c.d_state0) { TRY(c.d_state0.grow(c.state0.size())); c.state0_stale = true; }
  if (c.state0_stale) {   // on `stream` ahead of the launches that read it (render_device_run uploads before it forks the class streams)
    CU(cudaMemcpyAsync(c.d_state0, c.state0.data(), c.state0.size() * 4, cudaMemcpyHostToDevice, stream));
    CU(cudaStreamSynchronize(stream));   // c.state0 is pageable and changes with the next edit of a voice
    c.state0_stale = false;
  }
  *out = c.d_state0;
  return "";
}

// `l`: the words to run with. `reset_state`: the construction-time state that reset() restores (defaults to l.S).
std::string Bank::upload_voice(uint32_t voice, const Lowering& l, bool with_state, const std::vector<uint32_t>* reset_state) {
  TRY(rt_end_streak());
  uint32_t i = 0;
  if (VoiceClass* cp = locate(classes, voice, &i)) {
    VoiceClass& c = *cp;
    const uint32_t Vc = c.V();
    if (l.U != c.uniform || l.P.size() != c.np || l.S.size() != c.ns || (reset_state && reset_state->size() != c.ns))
      return "#U the voice does not fit its class: a class-uniform word (delay length, table, wave) or the word layout differs; rebuild the bank instead";
    if (with_state && c.form == Form::fdn) return "#U voices of a two-stage (FDN reverb) class cannot be replaced in place";
    TRY(sh_check(voice, l.shared));
    if (c.np) CU(cudaMemcpy2DAsync(c.d_params + i, (size_t)Vc * 4, l.P.data(), 4, 4, c.np, cudaMemcpyHostToDevice, stream));
    const std::vector<uint32_t> S0 = reset_state ? *reset_state : l.reset_image();
    for (uint32_t k = 0; k < c.ns; k++) c.state0[(size_t)k * Vc + i] = S0[k];
    c.state0_stale = true;
    if (with_state) {
      if (c.ns) CU(cudaMemcpy2DAsync(c.d_state + i, (size_t)Vc * 4, l.S.data(), 4, 4, c.ns, cudaMemcpyHostToDevice, stream));
      if (c.dl_floats) CU(cudaMemset2DAsync(c.d_dline + i, (size_t)Vc * 4, 0, 4, (size_t)c.dl_floats, stream));
    }
    CU(cudaStreamSynchronize(stream));  // `l` is pageable
    sh_uses[voice] = l.shared;
    return sh_rebuild();
  }
  return "internal: voice not found in any class";
}

std::string Bank::edit_event(uint32_t voice, double end_time, double fade_out) {
  if (voice >= V()) return "#A edit: voice index out of range";
  CU(cudaSetDevice(device));
  if (loop_arg > 0.0) return "#U edit: events of a looping sequencer are not edited on the device (their current times live in the state words)";
  if (!event_edit(nodes[voice].get(), end_time, fade_out)) return "#A edit: the voice is not a sequencer event";
  Lowering l;
  nodes[voice]->lower(l);
  if (!l.ok) return "#U " + l.why;
  return upload_voice(voice, l, false);
}

void Bank::lower_entering(HNode* n, Lowering* l0, Lowering* l, bool fading) const {
  n->set_sample_rate(unit_rate());
  n->lower(*l0);                                          // (a crossfading vertex lowers as ARRIVED: a bank reset leaves it at its second unit)
  const bool xf = fading && xfade_set_done(n, false);
  const bool ev = event_set_clock(n, seq_time);          // an event put into a running sequencer counts from now
  n->lower(*l);
  if (ev) event_set_clock(n, 0.0);
  if (xf) xfade_set_done(n, true);
}

std::string Bank::replace_voice(uint32_t voice, HNode* node) {
  std::unique_ptr<HNode> n(node);
  if (!n) return "#A replace: null node";
  if (voice >= V()) return "#A replace: voice index out of range";
  if (n->inputs() != nin || n->outputs() != nout) return "#U replace: the unit's arity differs from the bank's";
  CU(cudaSetDevice(device));
  std::string a, b;
  n->sig(a); nodes[voice]->sig(b);
  // another graph class (Net::replace takes any unit of the same arity, src/net.rs:460-470): the voice moves to the class of its new graph —
  // the classes are regrouped around it, every other voice keeps its running state (the slow path, like add_voice)
  slot_latest.erase(voice); xfade_latest.erase(voice);   // (a parked update belongs to the unit that leaves)
  if (a != b) return regroup(n.release(), (int)voice, nullptr);
  Lowering l0, l;
  lower_entering(n.get(), &l0, &l, false);
  if (!l.ok) return "#U " + l.why;
  const std::vector<uint32_t> S0 = l0.reset_image();
  TRY(upload_voice(voice, l, true, &S0));
  nodes[voice] = std::move(n);
  return "";
}

// Grow a running bank by one voice without disturbing the others: the running state and delay lines of every voice are read back,
// the classes are rebuilt with the new voice (it may found a new class: its program is compiled first, so a failure leaves the bank
// untouched), and the saved columns are written into the new layout. O(bank state) — the slow path behind push_event.
std::string Bank::add_voice(HNode* node, uint32_t* voice) { return regroup(node, -1, voice); }

// Net::remove on a bank made from a Net (src/net.rs:351-404: "connections from the unit are replaced with zeros"): the voice's place in the
// mix keeps its position and carries silence from now on.
std::string Bank::remove_voice(uint32_t voice) {
  if (voice >= V()) return "#A remove: voice index out of range";
  std::vector<float> z((size_t)nout, 0.0f);
  HNode* silent = mk_constant(nout, z.data());
  if (nin > 0) silent = mk_pipe(mk_sink(nin), silent);
  if (!silent) return "remove: could not build the silent unit";
  return replace_voice(voice, silent);
}

// `at` < 0: append the unit as a new voice (add_voice); else put it in place of voice `at` (replace_voice across classes).
std::string Bank::regroup(HNode* node, int at, uint32_t* voice, const Carry* carry) {
  std::unique_ptr<HNode> n(node);
  const char* what = at < 0 ? "add" : "replace";
  if (!n) return std::string("#A ") + what + ": null node";
  if (n->inputs() != nin || n->outputs() != nout) return std::string("#U ") + what + ": the unit's arity differs from the bank's";
  if (tree_mix && at < 0) return "#U add: a bank extracted from a Net mixes in the Net's order; rebuild it from the edited Net";
  for (auto& c : classes) if (c.form != Form::plain) return std::string("#U ") + what + ": banks with a two-stage class (FDN reverb, tensor-core convolver) cannot be regrouped in place; rebuild the bank";
  CU(cudaSetDevice(device));
  TRY(rt_end_streak());
  Lowering l0, l;
  lower_entering(n.get(), &l0, &l, true);
  if (!l.ok) return "#U " + l.why;
  { std::string sg, jerr; n->sig(sg); if (!get_program(sg, device, jerr)) return std::string("#U ") + what + ": no device program for `" + sg + "`: " + jerr; }
  // 1. read back what is running
  CU(cudaStreamSynchronize(stream));
  struct Saved { std::string sig; std::vector<uint32_t> uniform, voices, S; std::vector<float> D; uint32_t ns; uint64_t dl; };
  std::vector<Saved> saved;
  for (auto& c : classes) {
    Saved sv; sv.sig = c.sig; sv.uniform = c.uniform; sv.voices = c.voices; sv.ns = c.ns; sv.dl = c.dl_floats;
    sv.S.resize((size_t)c.ns * c.V()); sv.D.resize((size_t)c.dl_floats * c.V());
    if (!sv.S.empty()) CU(cudaMemcpy(sv.S.data(), c.d_state, sv.S.size() * 4, cudaMemcpyDeviceToHost));
    if (!sv.D.empty()) CU(cudaMemcpy(sv.D.data(), c.d_dline, sv.D.size() * 4, cudaMemcpyDeviceToHost));
    saved.push_back(std::move(sv));
  }
  const bool was_dirty = dirty; const double clock = seq_time;
  // 2. rebuild with the new voice (fresh state everywhere)
  uint32_t nv;
  if (at < 0) { nodes.push_back(std::move(n)); nv = V() - 1; }
  else { nv = (uint32_t)at; std::swap(nodes[nv], n); }        // `n` now holds the unit that leaves
  std::string e = lower_and_upload(true);
  if (!e.empty()) {
    if (at < 0) nodes.pop_back(); else std::swap(nodes[nv], n);
    std::string e2 = lower_and_upload(true);
    return std::string(what) + ": " + e + (e2.empty() ? " (the bank was rebuilt as it was; its running state is reset)" : " (and the bank could not be restored: " + e2 + ")");
  }
  // 3. put the saved columns back
  for (auto& c : classes) {
    const uint32_t Vc = c.V();
    std::vector<uint32_t> S = c.state0;
    std::vector<float> D((size_t)c.dl_floats * Vc, 0.0f);
    for (uint32_t i = 0; i < Vc; i++) {
      const uint32_t v = c.voices[i];
      uint32_t j = 0;
      if (v == nv) {   // the newcomer: live state (an event's clock = now); what reset() restores is its construction-time state
        const std::vector<uint32_t> S0 = l0.reset_image();
        for (uint32_t k = 0; k < c.ns && k < l.S.size(); k++) { S[(size_t)k * Vc + i] = l.S[k]; c.state0[(size_t)k * Vc + i] = S0[k]; }
        c.state0_stale = true;
        // a unit that keeps RUNNING inside the newcomer (the fading-out side of a crossfade): its words and delay lines move over
        if (const Saved* sv = carry ? locate(saved, v, &j) : nullptr) {
          const uint32_t Vo = (uint32_t)sv->voices.size();
          if (carry->src_s + carry->ns > sv->ns || carry->dst_s + carry->ns > c.ns || carry->src_d + carry->nd > sv->dl || carry->dst_d + carry->nd > c.dl_floats) return "internal: crossfade carry out of range";
          for (uint32_t k = 0; k < carry->ns; k++) S[(size_t)(carry->dst_s + k) * Vc + i] = sv->S[(size_t)(carry->src_s + k) * Vo + j];
          for (uint64_t q = 0; q < carry->nd; q++) D[(size_t)(carry->dst_d + q) * Vc + i] = sv->D[(size_t)(carry->src_d + q) * Vo + j];
        }
        continue;
      }
      if (const Saved* sv = locate(saved, v, &j)) {
        if (sv->sig != c.sig || sv->ns != c.ns || sv->dl != c.dl_floats) return "internal: a voice changed class while the bank grew";
        const uint32_t Vo = (uint32_t)sv->voices.size();
        for (uint32_t k = 0; k < c.ns; k++) S[(size_t)k * Vc + i] = sv->S[(size_t)k * Vo + j];
        for (uint64_t q = 0; q < c.dl_floats; q++) D[(size_t)q * Vc + i] = sv->D[(size_t)q * Vo + j];
      }
    }
    if (!S.empty()) CU(cudaMemcpyAsync(c.d_state, S.data(), S.size() * 4, cudaMemcpyHostToDevice, stream));
    if (!D.empty()) CU(cudaMemcpyAsync(c.d_dline, D.data(), D.size() * 4, cudaMemcpyHostToDevice, stream));
    CU(cudaStreamSynchronize(stream));
  }
  dirty = was_dirty; seq_time = clock;
  if (voice) *voice = nv;
  return "";
}

// Net::crossfade (src/net.rs:480-504) on a running bank: the voice becomes a vertex that fades from its unit to `unit` — of ANY graph class —
// over fade_time seconds (device: nodes.cuh Xfade<X, Y>, the arithmetic of src/vertex.rs:138-229) and is `unit` alone afterwards. The voice moves
// to the class Xfade<old, new> (compiled first if new); the old unit keeps running inside it: its state words and delay lines are carried over.
// A voice that has finished an earlier crossfade continues from its faded-in unit; while a fade is running the reference parks a further
// edit as `latest`: so does the bank (bank.h `xfade_latest`, `slot_service`).
std::string Bank::crossfade_voice(uint32_t voice, int ease, float fade_time, HNode* unit) {
  std::unique_ptr<HNode> n(unit);
  if (voice >= V()) return "#A crossfade: voice index out of range";
  if (!n || ease < 0 || ease > 1 || !(fade_time > 0.0f)) return "#A crossfade: needs a unit, fade 0 (Power) or 1 (Smooth) and a fade time > 0";
  if (n->inputs() != nin || n->outputs() != nout) return "#U crossfade: the unit's arity differs from the bank's";
  CU(cudaSetDevice(device));
  TRY(rt_end_streak());
  const HNode* cur = nodes[voice].get();
  Carry carry{0, 0, 0, 0, 0, 0};
  auto count = [](const HNode* h, uint32_t* ns, uint64_t* nd) { Lowering q; h->lower(q); *ns = (uint32_t)q.S.size(); *nd = 0; for (uint32_t d : q.dlen) *nd += d; return q.ok; };
  std::unique_ptr<HNode> old;
  if (const HNode* y = xfade_unit(cur, 1)) {   // the vertex crossfaded before: it must have arrived at its second unit
    uint32_t i = 0;
    if (const VoiceClass* c = locate(classes, voice, &i)) {
      CU(cudaStreamSynchronize(stream));
      uint32_t done = 0;
      CU(cudaMemcpy(&done, c->d_state + i, 4, cudaMemcpyDeviceToHost));   // state word 0 of Xfade: done
      if (!done) {
        // Vertex::enqueue with `next` occupied: the edit waits as `latest`, a newer one replaces it (src/vertex.rs:203-218). Its program — the
        // class Xfade<second unit, new unit> the voice will move to — is compiled now, so that a unit without a device program is refused here
        std::unique_ptr<HNode> probe(mk_xfade(y->clone(), n->clone(), ease, fade_time));
        std::string sg, jerr;
        if (!probe) return "#A crossfade: the units do not fit one vertex";
        probe->set_sample_rate(unit_rate());
        { Lowering q; probe->lower(q); if (!q.ok) return "#U " + q.why; }
        probe->sig(sg);
        if (!get_program(sg, device, jerr)) return "#U crossfade: no device program for `" + sg + "`: " + jerr;
        SlotLatest& w = xfade_latest[voice];
        w.unit = std::move(n); w.ease = ease; w.fade_time = (double)fade_time;
        return "";
      }
    }
    xfade_latest.erase(voice);
    uint32_t xs = 0; uint64_t xd = 0;
    if (!count(xfade_unit(cur, 0), &xs, &xd) || !count(y, &carry.ns, &carry.nd)) return "internal: crossfade: lowering failed";
    carry.src_s = 2u + xs; carry.src_d = xd;
    old.reset(y->clone());
  } else {
    if (!count(cur, &carry.ns, &carry.nd)) return "internal: crossfade: lowering failed";
    old.reset(cur->clone());
  }
  carry.dst_s = 2u; carry.dst_d = 0;      // Xfade<X, Y>: its own two state words, then X's, then Y's; X's delay lines first
  HNode* x = mk_xfade(old.release(), n.release(), ease, fade_time);
  if (!x) return "#A crossfade: the units do not fit one vertex";
  return regroup(x, (int)voice, nullptr, &carry);
}

// Slot::set on a live bank (src/slot.rs:64-71,124-151): the unit goes into the idle instance of the voice's Slot<X> and the device
// crossfades to it over fade_time seconds from the next block on. While a fade is running the update is parked as `latest` (see bank.h).
std::string Bank::slot_set(uint32_t voice, int ease, double fade_time, HNode* unit) {
  std::unique_ptr<HNode> n(unit);
  if (voice >= V()) return "#A slot: voice index out of range";
  if (!n || ease < 0 || ease > 1 || !(fade_time > 0.0)) return "#A slot: needs a unit, fade 0 (Power) or 1 (Smooth) and a fade time > 0";
  if (!is_slot(nodes[voice].get())) return "#A slot: the voice is not a slot (fdsp_slot)";
  return slot_arm_now(voice, ease, fade_time, n.release(), false);
}

std::string Bank::slot_arm_now(uint32_t voice, int ease, double fade_time, HNode* unit, bool force) {
  std::unique_ptr<HNode> n(unit);
  CU(cudaSetDevice(device));
  TRY(rt_end_streak());
  uint32_t i = 0;
  if (VoiceClass* cp = locate(classes, voice, &i)) {
    VoiceClass& c = *cp;
    const uint32_t Vc = c.V();
    if (c.form == Form::fdn || c.ns < 4 || ((c.ns - 4) & 1u) || (c.dl_floats & 1u)) return "slot: unexpected class layout";
    CU(cudaStreamSynchronize(stream));
    uint32_t head[2] = {0, 0};   // which, has_next of this voice
    CU(cudaMemcpy2D(head, 4, c.d_state + i, (size_t)Vc * 4, 4, 2, cudaMemcpyDeviceToHost));
    const bool fading = head[1] != 0 && !force;
    const int inst = (int)(head[0] ^ 1u);
    // arm a COPY of the voice's host slot: a refused unit leaves the host graph as it was (it replaces the original after the upload)
    std::unique_ptr<HNode> trial(nodes[voice]->clone());
    std::unique_ptr<HNode> parked(fading ? n->clone() : nullptr);   // a parked unit is checked now (with a copy), armed later
    if (!slot_arm(trial.get(), n.release(), inst, ease, fade_time)) return "#U slot: the unit's graph class differs from the slot's (same type expression needed)";
    Lowering l;
    trial->lower(l);
    if (!l.ok) return "#U " + l.why;
    if (l.U != c.uniform || l.P.size() != c.np || l.S.size() != c.ns) return "#U slot: the unit changes a class-uniform word (delay length, table, wave); rebuild the bank instead";
    TRY(sh_check(voice, l.shared));
    if (fading) {   // SlotBackend::handle_messages with `next` occupied: the update waits as `latest`, a newer one takes its place (:142-150)
      SlotLatest& w = slot_latest[voice];
      w.unit = std::move(parked); w.ease = ease; w.fade_time = fade_time;
      return "";
    }
    slot_latest.erase(voice);
    const uint32_t xs = (c.ns - 4) / 2, s0 = 4 + (uint32_t)inst * xs;
    const uint64_t xd = c.dl_floats / 2;
    CU(cudaMemcpy2DAsync(c.d_params + i, (size_t)Vc * 4, l.P.data(), 4, 4, c.np, cudaMemcpyHostToDevice, stream));
    if (xs) CU(cudaMemcpy2DAsync(c.d_state + (size_t)s0 * Vc + i, (size_t)Vc * 4, l.S.data() + s0, 4, 4, xs, cudaMemcpyHostToDevice, stream));
    if (xd) CU(cudaMemset2DAsync(c.d_dline + (size_t)inst * xd * Vc + i, (size_t)Vc * 4, 0, 4, (size_t)xd, stream));
    const uint32_t arm[3] = {1u, 0u, 0u};   // has_next = 1, fade_phase = 0.0
    CU(cudaMemcpy2DAsync(c.d_state + (size_t)1 * Vc + i, (size_t)Vc * 4, arm, 4, 4, 3, cudaMemcpyHostToDevice, stream));
    CU(cudaStreamSynchronize(stream));
    const std::vector<uint32_t> S0 = l.reset_image();
    for (uint32_t k = 0; k < c.ns; k++) c.state0[(size_t)k * Vc + i] = S0[k];   // reset() adopts the newest unit (:156-172)
    c.state0_stale = true;
    nodes[voice] = std::move(trial);
    sh_uses[voice] = l.shared;
    return sh_rebuild();
  }
  return "internal: voice not found in any class";
}

// Before a launch of n samples: a parked unit whose fade has ended is armed now (it starts fading with this launch's first block, the block
// after the one in which `next_phase` ran, src/slot.rs:163-172, src/vertex.rs:124-136); for the fades that are still running, the block in
// which each ends is found by replaying the device's per-block arithmetic (nodes.cuh Slot<X>::step in f64, Xfade<X, Y>::step in f32:
// phase_left, n_f, fade_phase += n_f / (fade_time sr)) from the voice's fade_phase word.
std::string Bank::slot_service(uint64_t n, uint64_t* cut) {
  *cut = n;
  // 1. arm what is ready. Arming a vertex regroups the classes, so the scan starts over after every arm.
  for (bool again = true; again;) {
    again = false;
    CU(cudaStreamSynchronize(stream));
    for (auto it = slot_latest.begin(); it != slot_latest.end(); ++it) {
      uint32_t i = 0; const VoiceClass* c = locate(classes, it->first, &i);
      if (!c || !is_slot(nodes[it->first].get())) { slot_latest.erase(it); again = true; break; }
      uint32_t has_next = 0;
      CU(cudaMemcpy(&has_next, c->d_state + (size_t)1 * c->V() + i, 4, cudaMemcpyDeviceToHost));
      if (has_next) continue;
      const uint32_t voice = it->first;
      SlotLatest w = std::move(it->second);
      slot_latest.erase(it);
      TRY(slot_arm_now(voice, w.ease, w.fade_time, w.unit.release(), false));
      again = true; break;
    }
    if (again) continue;
    for (auto it = xfade_latest.begin(); it != xfade_latest.end(); ++it) {
      uint32_t i = 0; const VoiceClass* c = locate(classes, it->first, &i);
      if (!c || !xfade_unit(nodes[it->first].get(), 1)) { xfade_latest.erase(it); again = true; break; }
      uint32_t done = 0;
      CU(cudaMemcpy(&done, c->d_state + i, 4, cudaMemcpyDeviceToHost));
      if (!done) continue;
      const uint32_t voice = it->first;
      SlotLatest w = std::move(it->second);
      xfade_latest.erase(it);
      TRY(crossfade_voice(voice, w.ease, (float)w.fade_time, w.unit.release()));
      again = true; break;
    }
  }
  // 2. where do the running fades with a parked unit end?
  auto consider = [&](uint64_t t_end) { if (t_end < *cut) *cut = t_end; };
  for (auto& kv : slot_latest) {
    uint32_t i = 0; const VoiceClass* c = locate(classes, kv.first, &i);
    if (!c) continue;
    uint32_t w[2] = {0, 0};
    CU(cudaMemcpy2D(w, 4, c->d_state + (size_t)2 * c->V() + i, (size_t)c->V() * 4, 4, 2, cudaMemcpyDeviceToHost));   // fade_phase (f64)
    double fade_time = 0.0, rate = 0.0;
    if (!slot_fade(nodes[kv.first].get(), &fade_time, &rate)) return "internal: a parked slot update on a voice that is not a slot";
    const uint64_t bits = ((uint64_t)w[1] << 32) | w[0];
    double phase; memcpy(&phase, &bits, 8);
    for (uint64_t t = 0; t < n;) {
      const int nb = (int)std::min<uint64_t>(64, n - t);
      const double span = fade_time * rate;
      const double left = (1.0 - phase) * span;
      const int phase_left = left > 0.0 ? (left < 1.0e9 ? (int)left : 1000000000) : 0;
      const int n_f = nb < phase_left ? nb : phase_left;
      phase += (double)n_f / (fade_time * rate);
      t += (uint64_t)nb;
      if (phase_left <= nb) { consider(t); break; }
    }
  }
  for (auto& kv : xfade_latest) {
    uint32_t i = 0; const VoiceClass* c = locate(classes, kv.first, &i);
    if (!c) continue;
    float phase = 0.0f;
    CU(cudaMemcpy(&phase, c->d_state + (size_t)1 * c->V() + i, 4, cudaMemcpyDeviceToHost));   // fade_phase (f32)
    float fade_time = 0.0f, rate = 0.0f;
    if (!xfade_fade(nodes[kv.first].get(), &fade_time, &rate)) return "internal: a parked crossfade on a voice that is not a crossfading vertex";
    for (uint64_t t = 0; t < n;) {
      const int nb = (int)std::min<uint64_t>(64, n - t);
      const float left = (1.0f - phase) * fade_time * rate;
      const int phase_left = left > 0.0f ? (left < 1.0e9f ? (int)left : 1000000000) : 0;
      const int n_f = nb < phase_left ? nb : phase_left;
      phase += (float)n_f / (fade_time * rate);
      t += (uint64_t)nb;
      if (phase_left <= nb) { consider(t); break; }
    }
  }
  return "";
}

std::string Bank::push_event(HNode* node, uint32_t* voice) {   // Sequencer::push on a running sequencer (src/sequencer.rs:319-360)
  std::unique_ptr<HNode> n(node);
  double s0, e0;
  if (!n || !event_times(n.get(), &s0, &e0)) return "#A push: not a sequencer event (fdsp_event)";
  if (loop_arg > 0.0) return "#U push: a looping sequencer bank takes its events before the first render";
  if (n->inputs() != nin || n->outputs() != nout) return "#U push: the event's arity differs from the bank's";
  CU(cudaSetDevice(device));
  const double sd = 1.0 / unit_rate();
  Lowering l0, l;
  lower_entering(n.get(), &l0, &l, false);   // (a start time in the past makes the event sound from the next block on)
  std::string want; n->sig(want);
  if (!l.ok) return "#U " + l.why;
  for (auto& c : classes) {
    if (c.sig != want || c.uniform != l.U || c.form == Form::fdn) continue;
    for (uint32_t v : c.voices) {
      if (!event_times(nodes[v].get(), &s0, &e0)) break;
      if (!(e0 <= seq_time + 0.5 * sd)) continue;   // Event::plan's end-of-event test at the start of the next block: still sounding
      const std::vector<uint32_t> S0 = l0.reset_image();
      TRY(upload_voice(v, l, true, &S0));
      nodes[v] = std::move(n);
      if (voice) *voice = v;
      return "";
    }
  }
  return "#N no finished event of the same graph class is free: create the bank with spare events of this class (finished, or ending at time 0), or rebuild it";
}

std::string Bank::reset() {  // AudioUnit::reset: back to the construction-time state
  CU(cudaSetDevice(device));
  TRY(rt_end_streak());
  while (!slot_latest.empty()) {   // SlotBackend::reset adopts the LATEST configuration (src/slot.rs:156-172): arm it (its words become the voice's reset image)
    auto it = slot_latest.begin();
    const uint32_t voice = it->first;
    SlotLatest w = std::move(it->second);
    slot_latest.erase(it);
    TRY(slot_arm_now(voice, w.ease, w.fade_time, w.unit.release(), true));
  }
  for (auto& c : classes) {
    // everything goes back to its construction-time value EXCEPT what the reference's reset leaves alone (keep_s / keep_d)
    const size_t Vc = c.V();
    { uint64_t at = 0;
      auto span = [&](uint64_t a, uint64_t b) -> cudaError_t { return b > a ? cudaMemcpyAsync(c.d_state + a * Vc, c.state0.data() + a * Vc, (size_t)(b - a) * Vc * 4, cudaMemcpyHostToDevice, stream) : cudaSuccess; };
      if (!c.state0.empty()) { for (auto& k : c.keep_s) { CU(span(at, k.first)); at = std::max(at, k.second); } CU(span(at, c.ns)); } }
    { uint64_t at = 0;
      auto span = [&](uint64_t a, uint64_t b) -> cudaError_t { return b > a ? cudaMemsetAsync(c.d_dline + a * Vc, 0, (size_t)(b - a) * Vc * sizeof(float), stream) : cudaSuccess; };
      if (c.dl_floats) { for (auto& k : c.keep_d) { CU(span(at, k.first)); at = std::max(at, k.second); } CU(span(at, c.dl_floats)); } }
    TRY(c.clear_history(stream));
  }
  CU(cudaStreamSynchronize(stream));
  dirty = false; seq_time = 0.0;
  for (auto& uses : sh_uses) for (auto& u : uses) if (u.kind == SH_TIMER) u.cell->set(0u);   // Timer::reset (src/shared.rs:223-226)
  return "";
}

// long launches of wavetable programs stage the table set in shared memory (TMA bulk copy, ~160 KB per CTA); short ones
// (process()-sized) read the tables through L1/L2 instead
static size_t table_bytes_of(const VoiceClass& c, uint32_t len) {
  const int wk = c.k ? c.k->wave_kind : -1;
  return (wk >= 0 && len >= 32u) ? device_wavetable(wk).data.size() * sizeof(float) : 0;   // at 64 samples the TMA-staged tables already win
}
// SMs of a device (the CTA shapes below are sized by it)
static uint32_t sm_count(int device) {
  static uint32_t n[64] = {};
  if (device < 0 || device >= 64) device = 0;
  if (!n[device]) { int v = 0; n[device] = cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && v > 0 ? (uint32_t)v : 1u; }
  return n[device];
}
// Stage-pipelined kernels (dsp/bank_kernel_st.cuh): programs with a heavy serial leaf (Moog ...) run their stages in different warps.
// Used for launches long enough to fill the pipeline and for classes too small to give every warp scheduler a voice-warp of its own
// (V <= SMs x 32: with a warp per scheduler already, stages only add hand-off work).
// FDSP_STAGED=0 switches them off (A/B).
static bool use_staged(const Program* k, uint32_t V, uint32_t len, uint32_t sms) {
  const char* e = getenv("FDSP_STAGED");            // read per call: the tests toggle it inside one process
  const int on = e ? atoi(e) : 1;
  return on != 0 && k && k->stages >= 2 && len >= 256u && V <= sms * 32u;
}
// CTAs (the rows of its partial mix), voices per CTA and kernel form of class c's voice program in a launch of len samples. Stage-pipelined:
// 32 voices per CTA while that still leaves SMs free, else 128 spread evenly (FDSP_STAGED_W=128 forces the wide shape: lets the tests reach
// it with few voices). Otherwise whole waves of CTAs with the voices spread evenly, but the dry stage of a two-stage class stays compact
// (few CTAs) so that it leaves the other SMs to the FDN kernel it is pipelined with.
struct ClassGrid { uint32_t ctas = 0, vpc = 0; bool staged = false; };
static ClassGrid class_grid(const VoiceClass& c, uint32_t len, int device) {
  ClassGrid g;
  if (!c.k) return g;
  const uint32_t V = c.V(), nsm = sm_count(device);
  const char* w = getenv("FDSP_STAGED_W");
  g.vpc = (uint32_t)c.k->threads;
  g.staged = use_staged(c.k.get(), V, len, nsm);
  if (g.staged && V <= nsm * 32u && !(w && atoi(w) == 128)) { g.vpc = 32u; g.ctas = (V + 31u) / 32u; }
  else if (g.staged) g.ctas = bank_grid(V, 128u, nsm, &g.vpc);
  else if (c.form == Form::fdn) g.ctas = (V + g.vpc - 1) / g.vpc;
  else g.ctas = bank_grid(V, g.vpc, nsm, &g.vpc);
  return g;
}

// ---- resident process() kernel
// A resident kernel holds a CTA (and, with staged wavetables, nearly all shared memory) on every SM: anything else launched on the device
// would sit behind it until its idle time-out. So at most one bank per device keeps one, and every entry point of EVERY bank of that
// device — they all begin with rt_stop() — first asks the owner to leave. (Banks of one device are driven from one thread at a time,
// like the units of the reference's audio thread; the registry itself is locked.)
std::string Bank::rt_stop() {
  Bank* other = nullptr;
  if (device >= 0 && device < 64) { std::lock_guard<std::mutex> lock(g_rt_mu); other = g_rt_owner[device]; if (other == this || (other && !other->rt_running)) other = nullptr; }
  if (other) TRY(other->rt_stop());
  if (!rt_running) return "";
  rt_ctl->doorbell = RT_QUIT;
  __sync_synchronize();
  rt_running = false;
  if (device >= 0 && device < 64) { std::lock_guard<std::mutex> lock(g_rt_mu); if (g_rt_owner[device] == this) g_rt_owner[device] = nullptr; }
  CU(cudaStreamSynchronize(stream));   // the kernel has saved the state words
  return "";
}
// One block through the resident kernel. `served` = false: the form does not apply (or the kernel had just left): the caller takes the
// one-launch-per-block path, which continues from the saved state.
std::string Bank::rt_process(uint32_t size, const float* in, float* out, bool* served) {
  *served = false;
#ifdef FDSP_HOST_EMUL
  (void)size; (void)in; (void)out; return "";
#else
  const char* rte = getenv("FDSP_RT");          // read per call: the tests toggle it inside one process
  const int on = rte ? atoi(rte) : 1;
  if (!on) { process_streak = 0; return ""; }
  if (has_parked()) { process_streak = 0; return ""; }   // parked Slot / crossfade updates are armed between launches (render_device)
  if (classes.size() != 1 || !(out_mode & 2u) || tree_mix || nout > 8 || nin > 8) return "";
  VoiceClass& c = classes[0];
  if (c.form != Form::plain || !c.k || !c.k->has_rt) return "";
  if (!sh_cells.empty()) return "";   // Shared controls are exchanged between calls, on the launch path (sh_pull / sh_push)
  uint32_t vpc = (uint32_t)c.k->threads;
  const uint32_t grid = bank_grid(c.V(), (uint32_t)c.k->threads, sm_count(device), &vpc);
  if (grid > sm_count(device)) return "";           // every CTA must be resident at once
  if (++process_streak < 3u && !rt_running) return "";   // a bank that is driven block by block: the third process() call in a row starts the kernel
  if (!rt_running) TRY(rt_stop());   // (another bank of this device may own the resident slot)
  TRY(rt_ctl.grow(1)); TRY(d_rt_relay.grow(4));
  TRY(d_rt_partial.grow((size_t)grid * nout * 64));
  if (!rt_running) {
    const uint32_t first = ++rt_seq; if (rt_seq >= 0xfffffff0u) rt_seq = 1;
    memset((void*)rt_ctl, 0, sizeof(RtCtl));
    rt_ctl->doorbell = first - 1u; rt_ctl->done = first - 1u;
    const uint32_t relay[4] = {first - 1u, 0u, 0u, 0u};
    CU(cudaMemcpyAsync(d_rt_relay, relay, 16, cudaMemcpyHostToDevice, stream));
    CU(cudaMemsetAsync(d_ticket, 0, 4, stream));
    BankArgs a;
    TRY(voice_args(c, 64, vpc, &a));
    a.partial = d_rt_partial; a.ticket = d_ticket;
    RtArgs rt{rt_ctl.dev(), d_rt_relay, first};
    CU(cudaStreamSynchronize(stream));   // the relay words are in place (pageable source)
    CU(c.k->launch_rt(a, rt, table_bytes_of(c, 64), stream));
    launches++;
    rt_running = true;
    if (device >= 0 && device < 64) { std::lock_guard<std::mutex> lock(g_rt_mu); g_rt_owner[device] = this; }
    rt_seq = first - 1u;
  }
  const uint32_t seq = ++rt_seq;
  if (nin > 0) { if (!in) return "#A bank has inputs but no input buffer was given"; memcpy((void*)rt_ctl->in, in, (size_t)nin * 64 * 4); }
  rt_ctl->size = size;
  __sync_synchronize();
  rt_ctl->doorbell = seq;
  const auto t_ring = std::chrono::steady_clock::now();
  for (uint64_t spins = 0;; spins++) {
    const uint32_t d = rt_ctl->done;
    if (d == seq) break;
    if (d == RT_EXITED) {                 // the kernel left (idle) just before the doorbell rang: not served, state saved
      rt_running = false; rt_seq--;
      CU(cudaStreamSynchronize(stream));
      return "";
    }
    if ((spins & 0xfffu) == 0xfffu && std::chrono::steady_clock::now() - t_ring > std::chrono::seconds(5)) {
      rt_ctl->doorbell = RT_QUIT; rt_running = false;
      return "process: the resident kernel does not answer (are all its CTAs resident? another kernel may hold the GPU)";
    }
    __builtin_ia32_pause();
  }
  __sync_synchronize();
  memcpy(out, (const void*)rt_ctl->out, (size_t)nout * 64 * 4);
  dirty = true; advance_clock(size);
  *served = true;
  return "";
#endif
}

std::string Bank::dom_mark(cudaStream_t st) {   // called in pairs: begin, end
  static const bool off = getenv("FDSP_NO_DOM") != nullptr;   // A/B: what the event records themselves cost
  if (!timing || off) return "";
  if (dom_n == dom_ev.size()) { Event e; CU(cudaEventCreate(e.put())); dom_ev.push_back(std::move(e)); }
  CU(cudaEventRecord(dom_ev[dom_n++], st));
  return "";
}

std::string Bank::render_device(uint64_t n, const float* in_dev, uint64_t in_stride, float* out_dev, uint64_t out_stride, float* mix_dev,
                                uint64_t mix_stride) {
  if (!has_parked()) return render_device_run(n, in_dev, in_stride, out_dev, out_stride, mix_dev, mix_stride);
  // parked Slot updates: the launch is cut behind the block in which a running fade ends, the parked unit is armed, the rest follows
  CU(cudaSetDevice(device));
  TRY(rt_stop());
  uint64_t done = 0;
  do {
    uint64_t cut = n - done;
    TRY(slot_service(n - done, &cut));
    if (cut == 0) break;
    TRY(render_device_run(cut, in_dev ? in_dev + done : nullptr, in_stride, out_dev ? out_dev + done : nullptr, out_stride, mix_dev ? mix_dev + done : nullptr, mix_stride));
    done += cut;
  } while (done < n);
  return "";
}

// The window (input, output rows, partial and fused mix) is the caller's: it is left empty here. state0 / dl_floats are the reset image of
// an Event class of a looping sequencer, null for every other class (state0_to_device); the kernels read dl_floats only with that image.
std::string Bank::voice_args(VoiceClass& c, uint32_t len, uint32_t vpc, BankArgs* a) {
  *a = BankArgs{};
  TRY(state0_to_device(c, &a->state0)); a->dl_floats = (uint32_t)c.dl_floats;
  a->params = c.d_params; a->state = c.d_state; a->uniform = c.d_uniform; a->dline = c.d_dline; a->wt = d_wt; a->row_map = c.d_rowmap;
  a->V = c.V(); a->n = len; a->vpc = vpc;
  a->sr = (float)sr; a->sd64 = (float)(1.0 / sr); a->sd32 = 1.0f / (float)sr;
  return "";
}

// One chunk of a render_device_run call, as its classes see it
struct Bank::Chunk {
  uint64_t t0, index; uint32_t len;
  bool want_v, want_m;                        // rows and partial mix wanted of the classes (a tree mix takes their rows and mixes them itself)
  float* out; uint32_t out_stride, out_t0;    // the rows: the caller's, or the tree mix's own from column 0
  float* mix; uint32_t mix_stride;
  bool pipelined;                             // two-stage classes run as a two-stream software pipeline
};
struct Bank::Pending { VoiceClass* c; Chunk w; int buf; };   // a partial-mix reduction of a pipelined class, issued one chunk late

static cudaError_t launch_program(const VoiceClass& c, const BankArgs& a, int mode, const ClassGrid& g, cudaStream_t st) {   // over a.n samples
  return g.staged ? c.k->launch_staged(a, mode, table_bytes_of(c, a.n), st) : c.k->launch(a, mode, table_bytes_of(c, a.n), st);
}

// the `grid` rows of a class's CTA-partial mix summed into the chunk's mix, or added to it (nothing when no mix is wanted)
std::string Bank::reduce_mix(const float* partial, uint32_t grid, const Chunk& w, bool accumulate, cudaStream_t st) {
  if (!w.want_m) return "";
  CU(launch_mix_reduce(partial, grid, (uint32_t)nout, w.len, w.mix, w.mix_stride, (uint32_t)w.t0, accumulate ? 1 : 0, st));
  launches++;
  return "";
}

// the deferred reductions (all, or those of class `only`), on `stream` behind the FDN kernel each one reads
std::string Bank::flush_pending(std::vector<Pending>& pending, const VoiceClass* only) {
  for (size_t q = 0; q < pending.size();) {
    Pending& pd = pending[q];
    if (only && pd.c != only) { q++; continue; }
    CU(cudaStreamWaitEvent(stream, pd.c->e_fdn[pd.buf], 0));
    TRY(reduce_mix(pd.buf ? pd.c->d_partial2 : pd.c->d_partial, pd.c->V(), pd.w, true, stream));
    pending.erase(pending.begin() + (long)q);
  }
  return "";
}

// stage 1 of a two-stage class, on `stream`: its program writes each voice's rows (d_dryrows) into `rows`, `stride` apart, from column `offset`
std::string Bank::launch_dry(VoiceClass& c, BankArgs d, const ClassGrid& g, float* rows, uint32_t stride, uint32_t offset) {
  d.out = rows; d.partial = nullptr; d.out_stride = stride; d.out_offset = offset; d.row_map = c.d_dryrows;
  CU(launch_program(c, d, 1, g, stream));
  launches++;
  return "";
}

// A plain class: its program, which finishes the mix-down itself in process()-sized launches (one launch instead of two), else the reduction
// of its partial mix. Concurrent classes run on their own streams; the caller reduces them once all are launched.
std::string Bank::run_plain(VoiceClass& c, const Chunk& w, const ClassGrid& g, BankArgs& a, bool first, bool concurrent) {
  const cudaStream_t ks = concurrent ? c.cstream : stream;
  const bool fused_mix = w.want_m && w.len <= 64;
  if (fused_mix) a.ticket = d_ticket;
  TRY(dom_mark(ks));
  CU(launch_program(c, a, (w.want_v ? 1 : 0) | (w.want_m ? 2 : 0), g, ks));
  TRY(dom_mark(ks));
  launches++;
  if (concurrent) CU(cudaEventRecord(c.e_done, ks));
  else if (!fused_mix) TRY(reduce_mix(c.d_partial, g.ctas, w, !first, stream));
  return "";
}

// An FDN class: the warp-per-voice reverb kernel on the rows of its dry stage, or on the bank's stereo input. Behind a dry stage in a
// pipelined call, stage 1 of chunk k runs on `stream` and stage 2 on `stream2`, the buffers alternate, and chunk k-1's partial mix is
// reduced after stage 1 of chunk k has been queued, so that the two stages of neighbouring chunks run side by side.
std::string Bank::run_fdn(VoiceClass& c, const Chunk& w, const ClassGrid& g, const BankArgs& a, bool first, std::vector<Pending>& pending) {
  const uint32_t V = c.V();
  if (w.len > TIME_CHUNK) return "internal: chunk";
  const bool pipe = w.pipelined && c.k;
  // voices (= warps) per CTA. Pipelined: leave SMs free for the CTAs of the dry stage of the next chunk (their shared-memory tables cannot
  // share an SM with an FDN CTA), otherwise the two stages serialise on SM residency
  const int cap = fdn_max_warps();
  const uint32_t nsm = sm_count(device);
  uint32_t sms = nsm;
  if (pipe) sms = g.ctas < nsm / 2 ? nsm - g.ctas : nsm / 2;
  int warps = (int)((V + sms - 1) / sms); if (warps > cap) warps = cap; if (warps < 1) warps = 1;
  FdnArgs f;
  f.params = c.d_params; f.state = c.d_state; f.uniform = c.d_uniform; f.p0 = c.p0; f.s0 = c.s0; f.u0 = c.u0; f.scalar_row = c.scalar_row;
  f.out = w.want_v ? w.out : nullptr; f.row_map = c.d_rowmap; f.out_stride = w.out_stride; f.out_offset = w.out_t0;
  f.partial = a.partial;
  f.ring = c.d_ring; f.ring_voice_stride = c.ring_floats; f.V = V; f.n = w.len;
  const int buf = (int)(w.index & 1);
  const bool solo = classes.size() == 1;
  cudaStream_t fs = stream;   // the FDN kernel's stream
  if (pipe) {
    float* dry = buf ? c.d_dry2 : c.d_dry;
    if (w.want_m && c.d_partial2.size() < (size_t)V * nout * w.len) TRY(c.d_partial2.grow((size_t)V * nout * PIPE_CHUNK));
    CU(cudaStreamWaitEvent(stream, c.e_fdn[buf], 0));   // FDN of chunk k-2 has consumed this dry buffer (no-op before the first record)
    TRY(launch_dry(c, a, g, dry, PIPE_CHUNK, 0));
    CU(cudaEventRecord(c.e_dry[buf], stream));
    // A bank of this one class keeps `stream` for the dry stage alone — chunk k + 1 follows chunk k with nothing in between, so it
    // holds its SMs before the wide FDN kernel of chunk k floods the rest — and reduces on stream2 behind the FDN kernel. With other
    // classes in the bank every reduction stays on `stream` (they accumulate into the same mix region), one chunk late.
    if (!solo) TRY(flush_pending(pending, &c));   // reduce chunk k-1 of this class (waits for its FDN)
    f.dry = dry; f.dry_voice_stride = 2ull * PIPE_CHUNK; f.dry_ch_stride = PIPE_CHUNK; f.dry_offset = 0;
    if (w.want_m && buf) f.partial = c.d_partial2;
    CU(cudaStreamWaitEvent(stream2, c.e_dry[buf], 0));
    fs = stream2;
  } else if (c.k) {  // stage 1: the fused dry program writes stereo rows [V][2][TIME_CHUNK]
    TRY(launch_dry(c, a, g, c.d_dry, TIME_CHUNK, 0));
    f.dry = c.d_dry; f.dry_voice_stride = 2ull * TIME_CHUNK; f.dry_ch_stride = TIME_CHUNK; f.dry_offset = 0;
  } else {    // reverb applied straight to the bank's stereo input
    f.dry = a.in; f.dry_voice_stride = 0; f.dry_ch_stride = a.in_stride; f.dry_offset = a.in_offset;
  }
  TRY(dom_mark(fs));
  CU(launch_fdn(f, warps, fs));
  TRY(dom_mark(fs));
  launches++;
  if (!pipe) return reduce_mix(c.d_partial, V, w, !first, stream);
  CU(cudaEventRecord(c.e_fdn[buf], stream2));
  if (!solo) pending.push_back({&c, w, buf});
  else TRY(reduce_mix(buf ? c.d_partial2 : c.d_partial, V, w, true, stream2));
  return "";
}

// A convolver class, on `stream`: the program in front of the convolver writes its rows behind the history columns; then x_lo, the
// Toeplitz GEMM tiles (rows straight into the caller's buffer, or an internal one), the history shift, and the voice-order fold of the rows
std::string Bank::run_conv(VoiceClass& c, const Chunk& w, const ClassGrid& g, const BankArgs& a) {
  const uint32_t V = c.V();
  TRY(launch_dry(c, a, g, c.d_cx, c.conv_stride, c.conv_H));
  CU(launch_conv_split(c.d_cx, c.d_cxl, V, c.conv_stride, c.conv_H, w.len, stream));
  float* y = w.want_v ? w.out : nullptr; uint32_t ys = w.out_stride, yo = w.out_t0;
  if (!y) {
    TRY(c.d_crows.grow((size_t)V * TIME_CHUNK));
    y = c.d_crows; ys = TIME_CHUNK; yo = 0;
  }
  TRY(dom_mark(stream));
  CU(launch_conv_tc(c.conv_maps, y, ys, yo, c.d_dryrows, V, w.len, c.conv_K, c.conv_H, stream));
  TRY(dom_mark(stream));
  CU(launch_conv_history(c.d_cx, c.d_cxl, V, c.conv_stride, c.conv_H, w.len, stream));
  launches += 3;
  if (w.want_m) { CU(launch_tree_mix(y, V, 1u, ys, yo, w.len, w.mix, w.mix_stride, (uint32_t)w.t0, 0, stream)); launches++; }
  return "";
}

std::string Bank::render_device_run(uint64_t n, const float* in_dev, uint64_t in_stride, float* out_dev, uint64_t out_stride, float* mix_dev,
                                    uint64_t mix_stride) {
  CU(cudaSetDevice(device));
  TRY(rt_stop());
  if (!in_process) process_streak = 0;
  if (nin > 0 && !in_dev) return "#A bank has inputs but no input buffer was given";
  const bool want_v = (out_mode & 1u) && out_dev, want_m = (out_mode & 2u) && mix_dev;
  if (!want_v && !want_m) return "#A no output buffer matches the bank's out_mode";
  if (n == 0) return "";
  if (in_stride > 0xffffffffull || out_stride > 0xffffffffull || mix_stride > 0xffffffffull) return "#A stride too large";
  if (timing) { CU(cudaEventRecord(ev0, stream)); dom_n = 0; }
  // Net-ordered mix: the voice kernels materialise per-voice rows (user buffer, or an internal one) and tree_mix_kernel adds
  // them in the Net's association order; the CTA-level partial mix is bypassed.
  const bool tree = tree_mix != 0 && want_m;
  // two-stage classes (fused dry program + warp-per-voice FDN) run as a two-stream software pipeline over PIPE_CHUNK samples
  bool pipelined = false;
  if (!tree && !getenv("FDSP_NO_PIPELINE")) for (auto& c : classes) pipelined = pipelined || c.fdn_with_dry();
  const uint32_t CH = tree ? 4096u : (pipelined ? PIPE_CHUNK : TIME_CHUNK);
  std::vector<Pending> pending;   // deferred CTA-partial reductions of pipelined classes (issued one chunk late, on `stream`)
  if (tree && !want_v) TRY(d_rows.grow((size_t)V() * nout * CH));
  // pipelined banks accumulate into a zeroed mix: cleared once for the whole call, so that nothing sits between the dry-stage launches of
  // consecutive chunks on `stream` (a gap there lets the wide FDN kernel of the previous chunk take every SM first)
  if (pipelined && want_m) CU(cudaMemset2DAsync(mix_dev, (size_t)mix_stride * 4, 0, (size_t)n * 4, (size_t)nout, stream));
  for (uint64_t t0 = 0, index = 0; t0 < n; t0 += CH, index++) {
    Chunk w;
    w.t0 = t0; w.index = index; w.len = (uint32_t)std::min<uint64_t>(CH, n - t0);
    w.mix = mix_dev; w.mix_stride = (uint32_t)mix_stride; w.pipelined = pipelined;
    w.want_v = want_v; w.want_m = want_m; w.out = out_dev; w.out_stride = (uint32_t)out_stride; w.out_t0 = (uint32_t)t0;
    if (tree) { w.want_m = false; if (!want_v) { w.want_v = true; w.out = d_rows; w.out_stride = CH; w.out_t0 = 0; } }
    bool first = !(pipelined && want_m);   // every class accumulates into the mix region zeroed above (reductions of pipelined classes arrive late)
    // several plain classes: launch the class kernels concurrently (own streams, forked from and joined back into `stream`); the
    // partial mixes are still reduced on `stream` in class order, so the result does not depend on how the kernels overlap
    bool concurrent = classes.size() > 1 && !pipelined && w.len > 64 && !getenv("FDSP_NO_CONCURRENT");
    for (auto& c : classes) concurrent = concurrent && c.form == Form::plain;
    for (auto& c : classes) { const uint32_t* s0 = nullptr; TRY(state0_to_device(c, &s0)); }   // (uploads stale reset images before the fork)
    if (concurrent) CU(cudaEventRecord(e_begin, stream));
    // (The classes start in class order: starting the one with the longest dependency chain first, on a high-priority stream, was worse for
    // config 5. Its CTAs hold ~195 KB of shared memory, so every light class then waits for all of it.)
    // Concurrent classes ask for ONE carve-out, the maximum: the class that stages the wavetables (~195 KB per CTA) needs it anyway, and kernels
    // that prefer different L1 / shared-memory splits do not share an SM.
    struct CarveGuard { int saved; CarveGuard() : saved(launch_carveout()) {} ~CarveGuard() { launch_carveout() = saved; } } carve_guard;
    if (concurrent) launch_carveout() = 100;
    for (auto& c : classes) {
      // every device operation of a bank is ordered on the bank's own streams: a class's stream is forked from `stream` and joined back below
      if (concurrent) {
        if (!c.cstream) { CU(cudaStreamCreateWithFlags(c.cstream.put(), cudaStreamNonBlocking)); CU(cudaEventCreateWithFlags(c.e_done.put(), cudaEventDisableTiming)); }
        CU(cudaStreamWaitEvent(c.cstream, e_begin, 0));
      }
      const ClassGrid g = class_grid(c, w.len, device);
      BankArgs a;
      TRY(voice_args(c, w.len, g.vpc, &a));
      a.in = in_dev; a.in_stride = (uint32_t)in_stride; a.in_offset = (uint32_t)t0;
      if (c.form != Form::conv) {   // the window of the programs that write rows and a partial mix
        if (w.want_m) {   // one row per CTA of a voice program, one per VOICE of the FDN kernel (its warps never meet); sized for TIME_CHUNK
          const uint32_t grid = c.form == Form::fdn ? c.V() : g.ctas;
          if (c.d_partial.size() < (size_t)grid * nout * w.len) TRY(c.d_partial.grow((size_t)grid * nout * TIME_CHUNK));
          a.partial = c.d_partial;
        }
        a.out = w.want_v ? w.out : nullptr; a.out_stride = w.out_stride; a.out_offset = w.out_t0;
        a.mix = w.mix; a.mix_stride = w.mix_stride; a.mix_offset = (uint32_t)t0; a.mix_accumulate = first ? 0 : 1;
        if (t0 > 0xffffffffull - TIME_CHUNK) return "#A render too long for one call";
      }
      switch (c.form) {
        case Form::plain: TRY(run_plain(c, w, g, a, first, concurrent)); break;
        case Form::fdn: TRY(run_fdn(c, w, g, a, first, pending)); break;
        case Form::conv: TRY(run_conv(c, w, g, a)); break;
      }
      if (!concurrent) first = false;
    }
    if (concurrent) for (auto& c : classes) {
      CU(cudaStreamWaitEvent(stream, c.e_done, 0));
      TRY(reduce_mix(c.d_partial, class_grid(c, w.len, device).ctas, w, !first, stream));
      first = false;
    }
    if (tree) {
      const size_t sc = tree_mix == 1 ? tree_mix_scratch_floats(V(), (uint32_t)nout, CH) : 0;   // balanced tree of a big bank: subtree sums first
      TRY(d_treepart.grow(sc));
      CU(launch_tree_mix(w.out, V(), (uint32_t)nout, w.out_stride, w.out_t0, w.len, mix_dev, (uint32_t)mix_stride, (uint32_t)t0, tree_mix == 1 ? 1 : 0, stream, sc ? d_treepart.get() : nullptr));
      launches += sc ? 2 : 1;
    }
  }
  TRY(flush_pending(pending, nullptr));   // also joins stream2 back into `stream`
  // a two-stage class alone in its bank reduces on stream2
  if (pipelined && classes.size() == 1) { CU(cudaEventRecord(e_begin, stream2)); CU(cudaStreamWaitEvent(stream, e_begin, 0)); }
  if (timing) CU(cudaEventRecord(ev1, stream));
  dirty = true; advance_clock(n);
  return "";
}

std::string Bank::ensure_staging(uint32_t chunk) {
  TRY(rt_stop());   // allocations synchronise with the device: no resident kernel may be waiting on its doorbell
  if (nin > 0) TRY(d_in.grow((size_t)nin * chunk));
  if (out_mode & 1u) TRY(d_out.grow((size_t)V() * nout * chunk));
  if (out_mode & 2u) TRY(d_mix.grow((size_t)nout * chunk));
  return "";
}

std::string Bank::render_host(uint64_t n, const float* in, float* out_voices, float* out_mix) {
  CU(cudaSetDevice(device));
  TRY(rt_stop());
  if (n == 0) return "";
  TRY(sh_pull());
  const size_t rows = (size_t)V() * nout;
  // chunk so that the per-voice staging buffer stays below ~512 MB
  uint32_t chunk = TIME_CHUNK;
  if ((out_mode & 1u) && out_voices) {
    const uint64_t cap = (512ull << 20) / (rows * 4);
    chunk = (uint32_t)std::max<uint64_t>(64, std::min<uint64_t>(TIME_CHUNK, cap / 64 * 64));
  }
  chunk = (uint32_t)std::min<uint64_t>(chunk, (n + 63) / 64 * 64);
  TRY(ensure_staging(chunk));
  for (uint64_t t0 = 0; t0 < n; t0 += chunk) {
    const uint32_t len = (uint32_t)std::min<uint64_t>(chunk, n - t0);
    if (nin > 0) {
      if (!in) return "#A bank has inputs but no input buffer was given";
      CU(cudaMemcpy2DAsync(d_in, (size_t)chunk * 4, in + t0, (size_t)n * 4, (size_t)len * 4, nin, cudaMemcpyHostToDevice, stream));
    }
    TRY(render_device(len, d_in, chunk, (out_voices ? d_out.get() : nullptr), chunk, (out_mix ? d_mix.get() : nullptr), chunk));
    if (out_voices && (out_mode & 1u)) CU(cudaMemcpy2DAsync(out_voices + t0, (size_t)n * 4, d_out, (size_t)chunk * 4, (size_t)len * 4, rows, cudaMemcpyDeviceToHost, stream));
    if (out_mix && (out_mode & 2u)) CU(cudaMemcpy2DAsync(out_mix + t0, (size_t)n * 4, d_mix, (size_t)chunk * 4, (size_t)len * 4, nout, cudaMemcpyDeviceToHost, stream));
  }
  CU(cudaStreamSynchronize(stream));
  return sh_push();
}

std::string Bank::process(uint32_t size, const float* in, float* out) {  // AudioUnit::process (size <= 64)
  if (size > 64) return "#A process: size must be <= 64 (MAX_BUFFER_SIZE)";
  if (size == 0) return "";
  CU(cudaSetDevice(device));
  {
    bool served = false;
    std::string re = rt_process(size, in, out, &served);
    if (!re.empty() || served) return re;
    const uint32_t keep = process_streak;
    re = rt_stop();                        // (no-op unless the resident kernel has just been declared unusable)
    if (!re.empty()) return re;
    process_streak = keep;
  }
  TRY(ensure_staging(64));
  const bool mix = (out_mode & 2u) != 0;  // mix mode wins for the AudioUnit surface; voices mode returns V*c channels
  const size_t rows = mix ? (size_t)nout : (size_t)V() * nout;
  TRY(h_in.grow((size_t)std::max(1, nin) * 64));
  TRY(h_out.grow(rows * 64));   // mapped: the mix is written straight into it by the GPU
  if (nin > 0) {
    if (!in) return "#A bank has inputs but no input buffer was given";
    memcpy(h_in, in, (size_t)nin * 64 * 4);
    CU(cudaMemcpyAsync(d_in, h_in, (size_t)nin * 64 * 4, cudaMemcpyHostToDevice, stream));
  }
  TRY(sh_pull());
  struct NoTiming { bool& t; explicit NoTiming(bool& x) : t(x) { t = false; } ~NoTiming() { t = true; } } no_timing(timing);  // no event records on this path
  struct InProcess { bool& f; explicit InProcess(bool& x) : f(x) { f = true; } ~InProcess() { f = false; } } in_proc(in_process);
  bool two_stage = false;   // pipelined classes clear / accumulate the mix region on the device: keep that in device memory
  for (auto& c : classes) two_stage = two_stage || c.fdn_with_dry();
  if (mix && two_stage) {
    TRY(render_device(size, d_in, 64, nullptr, 64, d_mix, 64));
    CU(cudaMemcpyAsync(h_out, d_mix, rows * 64 * 4, cudaMemcpyDeviceToHost, stream));
  } else if (mix) {
    // one block of mix is a few hundred bytes: mix_reduce_kernel stores it over PCIe into the mapped host buffer, which saves
    // the separate device-to-host copy of the latency-critical process() path
    TRY(render_device(size, d_in, 64, nullptr, 64, h_out.dev(), 64));
  } else {
    TRY(render_device(size, d_in, 64, d_out, 64, nullptr, 64));
    CU(cudaMemcpyAsync(h_out, d_out, rows * 64 * 4, cudaMemcpyDeviceToHost, stream));
  }
  CU(cudaStreamSynchronize(stream));
  memcpy(out, h_out, rows * 64 * 4);
  return sh_push();
}

std::string Bank::clone_into(Bank& dst) const {
  TRY(const_cast<Bank*>(this)->rt_stop());
  std::vector<HNode*> copies;
  for (auto& n : nodes) copies.push_back(n->clone());
  dst.sr = sr; dst.tree_mix = tree_mix; dst.net_rate = net_rate; dst.vertex_of_voice = vertex_of_voice;
  TRY(dst.init(copies, device, out_mode));
  for (auto& n : dst.nodes) n->set_sample_rate(sr);
  TRY(dst.lower_and_upload(true));
  CU(cudaSetDevice(device));
  // the running state is copied on the source's stream, behind its renders and ahead of its next one; the clone's stream waits for it
  auto copy = [&](void* d, const void* s, size_t bytes) { return cudaMemcpyAsync(d, s, bytes, cudaMemcpyDeviceToDevice, stream); };
  for (size_t i = 0; i < classes.size(); i++) {
    const VoiceClass& s = classes[i]; VoiceClass& d = dst.classes[i];
    if (!s.state0.empty()) CU(copy(d.d_state, s.d_state, s.state0.size() * 4));
    if (s.dl_floats) CU(copy(d.d_dline, s.d_dline, (size_t)s.dl_floats * s.V() * 4));
    if (s.ring_floats && s.d_ring && d.d_ring) CU(copy(d.d_ring, s.d_ring, (size_t)s.ring_floats * s.V() * 4));
    if (s.form == Form::conv && d.form == Form::conv) { CU(copy(d.d_cx, s.d_cx, (size_t)s.V() * s.conv_stride * 4)); CU(copy(d.d_cxl, s.d_cxl, (size_t)s.V() * s.conv_stride * 4)); }
  }
  CU(cudaEventRecord(dst.e_begin, stream));
  CU(cudaStreamWaitEvent(dst.stream, dst.e_begin, 0));
  dst.dirty = dirty; dst.seq_time = seq_time;
  for (auto& kv : slot_latest) { SlotLatest& w = dst.slot_latest[kv.first]; w.unit.reset(kv.second.unit->clone()); w.ease = kv.second.ease; w.fade_time = kv.second.fade_time; }
  for (auto& kv : xfade_latest) { SlotLatest& w = dst.xfade_latest[kv.first]; w.unit.reset(kv.second.unit->clone()); w.ease = kv.second.ease; w.fade_time = kv.second.fade_time; }
  return "";
}

// ---- Shared controls
namespace {
std::string cell_name(const SharedCell* c) { char b[40]; snprintf(b, sizeof b, "%p", (const void*)c); return std::string("the Shared at ") + b; }
}
std::string Bank::sh_check(uint32_t voice, const std::vector<SharedUse>& uses) const {
  std::map<const SharedCell*, int> how;   // bit 0 read, bit 1 written
  for (size_t v = 0; v < sh_uses.size(); v++)
    for (auto& u : (v == voice ? uses : sh_uses[v])) how[u.cell] |= u.kind == SH_READ ? 1 : 2;
  if (sh_uses.empty()) for (auto& u : uses) how[u.cell] |= u.kind == SH_READ ? 1 : 2;
  for (auto& kv : how)
    if (kv.second == 3) return "#U " + cell_name(kv.first) + " is both read (var / var_fn) and written (monitor / timer) in one bank: what a voice reads would depend on the voice order inside a block";
  return "";
}

std::string Bank::sh_rebuild() {
  std::map<const SharedCell*, int> index;
  sh_cells.clear(); sh_last.clear(); sh_last_writer.clear();
  size_t stage = 0;
  auto cell_of = [&](SharedCell* c) { auto it = index.find(c); if (it != index.end()) return it->second; const int k = (int)sh_cells.size(); index[c] = k; sh_cells.emplace_back(c); sh_last_writer.emplace_back(); return k; };
  for (size_t ci = 0; ci < classes.size(); ci++) {
    VoiceClass& c = classes[ci];
    const uint32_t Vc = c.V();
    c.sh_rows.clear(); c.sh_cell.clear(); c.sh_img.clear();
    std::map<uint32_t, size_t> row;
    for (uint32_t i = 0; i < Vc; i++)
      for (auto& u : sh_uses[c.voices[i]]) {
        const int k = cell_of(u.cell);
        if (u.kind != SH_READ) {   // the last voice in bank order, and within it the last writer in evaluation order
          ShWriter& w = sh_last_writer[k];
          if (w.cls < 0 || c.voices[i] >= w.voice) { w.cls = (int)ci; w.word = u.word; w.col = i; w.voice = c.voices[i]; }
          continue;
        }
        auto it = row.find(u.word);
        if (it == row.end()) { it = row.emplace(u.word, c.sh_rows.size()).first; c.sh_rows.push_back(u.word); c.sh_cell.resize(c.sh_rows.size() * Vc, -1); }
        c.sh_cell[it->second * Vc + i] = k;
      }
    if (c.sh_rows.empty()) continue;
    // the image starts from what the device holds: a row can mix readers with other voices' plain parameter words
    c.sh_img.resize(c.sh_rows.size() * Vc);
    stage += c.sh_img.size();
    CU(cudaStreamSynchronize(stream));
    for (size_t r = 0; r < c.sh_rows.size(); r++) CU(cudaMemcpy(c.sh_img.data() + r * Vc, c.d_params + (size_t)c.sh_rows[r] * Vc, (size_t)Vc * 4, cudaMemcpyDeviceToHost));
  }
  if (stage > sh_stage.size() && sh_pending) { CU(cudaEventSynchronize(sh_copied)); sh_pending = false; }   // (grow frees the staging)
  TRY(sh_stage.grow(stage));
  if (stage && !sh_copied) CU(cudaEventCreateWithFlags(sh_copied.put(), cudaEventDisableTiming));
  return "";
}

std::string Bank::sh_pull() {
  if (sh_cells.empty()) return "";
  std::vector<uint32_t> now(sh_cells.size());
  for (size_t k = 0; k < now.size(); k++) now[k] = sh_cells[k].c->get();   // one snapshot for the whole call
  if (now == sh_last) return "";
  CU(cudaSetDevice(device));
  if (sh_pending) { CU(cudaEventSynchronize(sh_copied)); sh_pending = false; }   // (the previous call's row copies: long done by now)
  size_t at = 0;
  for (auto& c : classes) {
    const uint32_t Vc = c.V();
    for (size_t r = 0; r < c.sh_rows.size(); r++, at += Vc) {
      bool changed = false;
      for (uint32_t i = 0; i < Vc; i++) {
        const int32_t k = c.sh_cell[r * Vc + i];
        if (k >= 0 && c.sh_img[r * Vc + i] != now[k]) { c.sh_img[r * Vc + i] = now[k]; changed = true; }
      }
      if (!changed) continue;
      if (at + Vc > sh_stage.size()) return "internal: Shared staging too small";
      memcpy(sh_stage + at, c.sh_img.data() + r * Vc, (size_t)Vc * 4);
      CU(cudaMemcpyAsync(c.d_params + (size_t)c.sh_rows[r] * Vc, sh_stage + at, (size_t)Vc * 4, cudaMemcpyHostToDevice, stream));
      sh_pending = true;
    }
  }
  if (sh_pending) CU(cudaEventRecord(sh_copied, stream));
  sh_last = std::move(now);
  return "";
}

std::string Bank::sh_push() {
  if (!sh_writes()) return "";
  CU(cudaSetDevice(device));
  CU(cudaStreamSynchronize(stream));
  for (size_t k = 0; k < sh_cells.size(); k++) {
    const ShWriter& w = sh_last_writer[k];
    if (w.cls < 0) continue;
    const VoiceClass& c = classes[(size_t)w.cls];
    uint32_t word = 0;
    CU(cudaMemcpy(&word, c.d_state + (size_t)w.word * c.V() + w.col, 4, cudaMemcpyDeviceToHost));
    sh_cells[k].c->set(word);
  }
  return "";
}

}  // namespace host
}  // namespace fdsp

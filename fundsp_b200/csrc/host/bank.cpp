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
// sub-chunk of two-stage (dry program -> FDN reverb) classes: stage 1 of chunk k+1 overlaps stage 2 of chunk k (FDSP_PIPE_CHUNK: tuning)
static uint32_t pipe_chunk() {
  static const uint32_t v = [] { const char* e = getenv("FDSP_PIPE_CHUNK"); uint32_t x = e ? (uint32_t)atoi(e) : 2048u; x = x / 64u * 64u; return x < 256u ? 256u : (x > TIME_CHUNK ? TIME_CHUNK : x); }();
  return v;
}
#define PIPE_CHUNK pipe_chunk()

std::string cuerr(const char* what, cudaError_t e) { return std::string(what) + ": " + cudaGetErrorString(e); }
#define CU(call)                                          \
  do {                                                    \
    cudaError_t e_ = (call);                              \
    if (e_ != cudaSuccess) return cuerr(#call, e_);       \
  } while (0)

template <class T> std::string dev_alloc(T** p, size_t count) {
  if (*p) { cudaFree(*p); *p = nullptr; }
  if (count == 0) return "";
  CU(cudaMalloc((void**)p, count * sizeof(T)));
  return "";
}
}  // namespace

// `Pipe<X, Convolver>` with a response long enough for 128-wide tiles goes to the tensor-core form (FDSP_TC_CONV=0: direct form only;
// FDSP_TC_MINK: shortest response, default 32 taps). One output channel, and not on the CPU mock device.
static bool tc_conv_wanted(const std::string& sig, const Lowering& l, int nout) {
#ifdef FDSP_HOST_EMUL
  (void)sig; (void)l; (void)nout; return false;
#else
  static const std::string CT = ",Convolver>";
  const char* e = getenv("FDSP_TC_CONV"); const char* m = getenv("FDSP_TC_MINK");
  if (e && atoi(e) == 0) return false;
  const uint32_t mink = m ? (uint32_t)atoi(m) : 32u;
  return nout == 1 && sig.compare(0, 5, "Pipe<") == 0 && sig.size() > 5 + CT.size() && sig.compare(sig.size() - CT.size(), CT.size(), CT) == 0 && l.conv_K >= mink &&
         l.conv_off + 2u + l.conv_K == l.U.size();
#endif
}

namespace {
std::mutex g_rt_mu;          // registry of the bank that owns each device's resident process() kernel (see rt_stop)
Bank* g_rt_owner[64] = {};
}
Bank::~Bank() {
  cudaSetDevice(device);
  rt_stop();
  if (device >= 0 && device < 64) { std::lock_guard<std::mutex> lock(g_rt_mu); if (g_rt_owner[device] == this) g_rt_owner[device] = nullptr; }
  if (rt_ctl) cudaFreeHost(rt_ctl);
  cudaFree(d_rt_relay); cudaFree(d_rt_partial);
  for (auto& c : classes) {
    cudaFree(c.d_params); cudaFree(c.d_state); cudaFree(c.d_state0); cudaFree(c.d_uniform); cudaFree(c.d_rowmap); cudaFree(c.d_dline); cudaFree(c.d_partial); cudaFree(c.d_ring); cudaFree(c.d_dry); cudaFree(c.d_dryrows); cudaFree(c.d_dry2); cudaFree(c.d_partial2); cudaFree(c.d_cx); cudaFree(c.d_cxl); cudaFree(c.d_th); cudaFree(c.d_tl); cudaFree(c.d_crows); for (int q = 0; q < 2; q++) { if (c.e_dry[q]) cudaEventDestroy(c.e_dry[q]); if (c.e_fdn[q]) cudaEventDestroy(c.e_fdn[q]); } if (c.cstream) cudaStreamDestroy(c.cstream); if (c.e_done) cudaEventDestroy(c.e_done);
  }
  for (float* p : d_wtdata) cudaFree(p);
  cudaFree(d_wt); cudaFree(d_in); cudaFree(d_out); cudaFree(d_mix); cudaFree(d_rows); cudaFree(d_treepart);
  if (h_in) cudaFreeHost(h_in);
  if (h_out) cudaFreeHost(h_out);
  for (cudaEvent_t e : dom_ev) cudaEventDestroy(e);
  if (ev0) cudaEventDestroy(ev0);
  if (ev1) cudaEventDestroy(ev1);
  if (e_begin) cudaEventDestroy(e_begin);
  cudaFree(d_ticket);
  if (stream2) cudaStreamDestroy(stream2);
  if (stream) cudaStreamDestroy(stream);
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
  { std::string re = rt_stop(); if (!re.empty()) return re; }   // (another bank's resident process() kernel would make the allocations below wait for its idle time-out)
  // `stream` carries the latency-bound voice programs (few CTAs, long serial chains) and gets the highest priority, so that in
  // the two-stage pipeline its CTAs are placed before the wide FDN kernel of the previous chunk (stream2) fills every SM.
  int prio_lo = 0, prio_hi = 0;
  CU(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
  CU(cudaStreamCreateWithPriority(&stream, cudaStreamNonBlocking, prio_hi));
  CU(cudaStreamCreateWithPriority(&stream2, cudaStreamNonBlocking, prio_lo));
  CU(cudaEventCreate(&ev0)); CU(cudaEventCreate(&ev1)); CU(cudaEventCreateWithFlags(&e_begin, cudaEventDisableTiming));
  CU(cudaMalloc((void**)&d_ticket, 4)); CU(cudaMemset(d_ticket, 0, 4));
  return lower_and_upload(true);
}

std::string Bank::lower_and_upload(bool upload_state) {
  CU(cudaSetDevice(device));
  { std::string re = rt_stop(); if (!re.empty()) return re; } process_streak = 0;
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
      const uint32_t nu_static = c.nu - lo.l.extraU;   // what the device templates count (NU); the rest is variable-length uniform data
      std::string jerr, prog_sig = lo.sig;
      // reverb_stereo tail -> warp-per-voice FDN kernel; the part in front of it (if any) stays a fused per-voice program
      static const std::string REV = "Pipe<Pipe<MultiSplit<2,16>,Feedback<1,Multi<30,0,32,Pipe<Delay,Fir<3>>>>>,Binop<2,Multi<31,0,32,Panner<1>>,Constant<2>>>";
      const std::string wet_tail = ",Bus<MultiPass<2>,Unop<3," + REV + ">>>", pipe_tail = "," + REV + ">";
      auto ends_with = [](const std::string& s, const std::string& t) { return s.size() >= t.size() && s.compare(s.size() - t.size(), t.size(), t) == 0; };
      bool wet = false;
      const bool fdn_off = getenv("FDSP_DISABLE_FDN") != nullptr;  // A/B switch: run reverbs in the generic thread-per-voice form
      if (fdn_off) {}
      else if (lo.sig == REV && nin == 2) { c.fdn = true; prog_sig.clear(); }
      else if (lo.sig == "Bus<MultiPass<2>,Unop<3," + REV + ">>" && nin == 2) { c.fdn = true; wet = true; prog_sig.clear(); }   // dry + g * reverb on a stereo bus
      else if (lo.sig.compare(0, 5, "Pipe<") == 0 && ends_with(lo.sig, wet_tail)) { c.fdn = true; wet = true; prog_sig = lo.sig.substr(5, lo.sig.size() - 5 - wet_tail.size()); }
      else if (lo.sig.compare(0, 5, "Pipe<") == 0 && ends_with(lo.sig, pipe_tail)) { c.fdn = true; prog_sig = lo.sig.substr(5, lo.sig.size() - 5 - pipe_tail.size()); }
      if (c.fdn) {
        for (size_t k = lo.l.U.size() - 32; k < lo.l.U.size(); k++) if (lo.l.U[k] < FDN_MIN_RING) c.fdn = false;  // the kernel's prefetch distance needs every delay >= 192 samples
        if (!c.fdn) prog_sig = lo.sig;
      }
      if (c.fdn) {
        c.p0 = c.np - 162; c.s0 = c.ns - 160; c.u0 = c.nu - 32;
        c.scalar_row = wet ? (int)c.p0 - 1 : -1;
        for (size_t k = 0; k < lo.l.dlen.size(); k++) { if (k + 32 >= lo.l.dlen.size()) c.ring_floats += fdn_ring_phys(lo.l.dlen[k]); else c.dl_floats += lo.l.dlen[k]; }
        if (!prog_sig.empty()) {
          c.k = get_program(prog_sig, device, jerr);
          if (!c.k) return "#U no device program for the dry stage `" + prog_sig + "`: " + jerr;
          if ((uint32_t)c.k->NP != c.p0 - (wet ? 1u : 0u) - lo.l.extraP || (uint32_t)c.k->NS != c.s0 || (uint32_t)c.k->NU != c.u0 - lo.l.extraU || c.k->IN != nin || c.k->OUT != 2)
            return "internal: dry-stage layout of `" + prog_sig + "` disagrees with the host lowering";
        }
      } else if (tc_conv_wanted(lo.sig, lo.l, nout)) {
        // `X >> convolve(h)`: X stays a fused per-voice program that writes its rows, the tap contraction runs on tensor cores. The
        // Convolver's own words (ring index, history ring) stay in the layout and are simply not used by this form.
        static const std::string CT = ",Convolver>";
        const std::string xsig = lo.sig.substr(5, lo.sig.size() - 5 - CT.size());
        for (uint32_t d : lo.l.dlen) c.dl_floats += d;
        c.k = get_program(xsig, device, jerr);
        if (!c.k) return "#U no device program for `" + xsig + "` (in front of the convolver): " + jerr;
        if ((uint32_t)c.k->NP != c.np - lo.l.extraP || (uint32_t)c.k->NS + 1u != c.ns || (uint32_t)c.k->NU + 2u != nu_static || c.k->IN != nin || c.k->OUT != 1)
          return "internal: layout of `" + xsig + "` in front of the convolver disagrees with the host lowering";
        c.conv = true; c.conv_K = lo.l.conv_K; c.conv_off = lo.l.conv_off;
        c.conv_H = (c.conv_K - 1u + 31u) / 32u * 32u; if (c.conv_H == 0) c.conv_H = 32;
        c.conv_J = conv_tc_toeplitz_cols(c.conv_K); c.conv_stride = c.conv_H + TIME_CHUNK;
      } else {
        for (uint32_t d : lo.l.dlen) c.dl_floats += d;
        c.k = get_program(lo.sig, device, jerr);
        if (!c.k) return "#U no device program for graph class `" + lo.sig + "`: " + jerr;
        if ((uint32_t)c.k->NP != c.np - lo.l.extraP || (uint32_t)c.k->NS != c.ns || (uint32_t)c.k->NU != nu_static || c.k->IN != nin || c.k->OUT != nout)
          return "internal: host lowering of `" + lo.sig + "` disagrees with the device word layout";
      }
      {   // reset exemptions of this graph class, in the class's own word / delay-line coordinates
        for (auto& r : lo.l.keepS) if (r.second > r.first) c.keep_s.emplace_back(r.first, r.second);
        std::vector<uint64_t> doff(lo.l.dlen.size() + 1, 0);
        const size_t nd_lines = c.fdn ? lo.l.dlen.size() - 32 : lo.l.dlen.size();   // the last 32 lines of an FDN class live in its rings
        for (size_t k = 0; k < lo.l.dlen.size(); k++) doff[k + 1] = doff[k] + (k < nd_lines ? lo.l.dlen[k] : 0u);
        for (auto& r : lo.l.keepD) if (r.second > r.first && r.second <= nd_lines) c.keep_d.emplace_back(doff[r.first], doff[r.second]);
        std::sort(c.keep_s.begin(), c.keep_s.end()); std::sort(c.keep_d.begin(), c.keep_d.end());
      }
      fresh.push_back(std::move(c));
    } else ci = it->second;
    fresh[ci].voices.push_back((uint32_t)v);
    std::string().swap(lo.key); std::vector<uint32_t>().swap(lo.l.U);   // the class keeps the uniform words (a sampler voice's may be a whole wave)
  }
  if (fresh.size() > 1) {   // the tensor-core convolver form is for one-class banks (its mix-down is the voice-order fold of its own rows)
    for (auto& c : fresh) if (c.conv) {
      std::string jerr;
      c.conv = false;
      c.k = get_program(c.sig, device, jerr);
      if (!c.k) return "#U no device program for graph class `" + c.sig + "`: " + jerr;
    }
  }
  // 2. keep device buffers of classes that survive unchanged (same key order / sizes), else rebuild
  const bool same_shape = classes.size() == fresh.size() && std::equal(classes.begin(), classes.end(), fresh.begin(), [](const VoiceClass& a, const VoiceClass& b) {
                            return a.sig == b.sig && a.voices == b.voices && a.uniform == b.uniform; });
  if (!same_shape) {
    for (auto& c : classes) { cudaFree(c.d_params); cudaFree(c.d_state); cudaFree(c.d_state0); cudaFree(c.d_uniform); cudaFree(c.d_rowmap); cudaFree(c.d_dline); cudaFree(c.d_partial); cudaFree(c.d_ring); cudaFree(c.d_dry); cudaFree(c.d_dryrows); cudaFree(c.d_dry2); cudaFree(c.d_partial2); cudaFree(c.d_cx); cudaFree(c.d_cxl); cudaFree(c.d_th); cudaFree(c.d_tl); cudaFree(c.d_crows); for (int q = 0; q < 2; q++) { if (c.e_dry[q]) cudaEventDestroy(c.e_dry[q]); if (c.e_fdn[q]) cudaEventDestroy(c.e_fdn[q]); } if (c.cstream) cudaStreamDestroy(c.cstream); if (c.e_done) cudaEventDestroy(c.e_done); }
    classes = std::move(fresh);
    upload_state = true;
  }
  for (auto& c : classes) {
    const uint32_t V = c.V(); const int NP = (int)c.np, NS = (int)c.ns;
    std::vector<uint32_t> P((size_t)NP * V), S((size_t)NS * V), rows(V);
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
      std::string e;
      if (!(e = dev_alloc(&c.d_params, P.size())).empty()) return e;
      if (!(e = dev_alloc(&c.d_state, S.size())).empty()) return e;
      if (!(e = dev_alloc(&c.d_uniform, c.uniform.size())).empty()) return e;
      if (!(e = dev_alloc(&c.d_rowmap, rows.size())).empty()) return e;
      if (!(e = dev_alloc(&c.d_dline, (size_t)c.dl_floats * V)).empty()) return e;
      if (c.fdn) {
        if (!(e = dev_alloc(&c.d_ring, (size_t)c.ring_floats * V)).empty()) return e;
        if (c.k) {
          if (!(e = dev_alloc(&c.d_dry, (size_t)V * 2 * TIME_CHUNK)).empty()) return e;
          if (!(e = dev_alloc(&c.d_dry2, (size_t)V * 2 * PIPE_CHUNK)).empty()) return e;
          for (int q = 0; q < 2; q++) { CU(cudaEventCreateWithFlags(&c.e_dry[q], cudaEventDisableTiming)); CU(cudaEventCreateWithFlags(&c.e_fdn[q], cudaEventDisableTiming)); }
          if (!(e = dev_alloc(&c.d_dryrows, V)).empty()) return e;
          std::vector<uint32_t> id(V);
          for (uint32_t i = 0; i < V; i++) id[i] = 2 * i;
          CU(cudaMemcpy(c.d_dryrows, id.data(), V * 4, cudaMemcpyHostToDevice));
        }
      }
      if (c.conv) {
        if (!(e = dev_alloc(&c.d_cx, (size_t)V * c.conv_stride)).empty()) return e;
        if (!(e = dev_alloc(&c.d_cxl, (size_t)V * c.conv_stride)).empty()) return e;
        if (!(e = dev_alloc(&c.d_th, (size_t)128 * c.conv_J)).empty()) return e;
        if (!(e = dev_alloc(&c.d_tl, (size_t)128 * c.conv_J)).empty()) return e;
        if (!(e = dev_alloc(&c.d_dryrows, V)).empty()) return e;
        std::vector<uint32_t> id(V);
        for (uint32_t i = 0; i < V; i++) id[i] = i;
        CU(cudaMemcpy(c.d_dryrows, id.data(), V * 4, cudaMemcpyHostToDevice));
        CU(conv_tc_make_maps(c.d_cx, c.d_cxl, V, c.conv_stride, c.d_th, c.d_tl, c.conv_J, &c.conv_maps));
      }
      CU(cudaMemcpy(c.d_rowmap, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice));
      if (!c.uniform.empty()) CU(cudaMemcpy(c.d_uniform, c.uniform.data(), c.uniform.size() * 4, cudaMemcpyHostToDevice));
    }
    if (!P.empty()) CU(cudaMemcpy(c.d_params, P.data(), P.size() * 4, cudaMemcpyHostToDevice));
    if (upload_state) {
      if (!S.empty()) CU(cudaMemcpy(c.d_state, S.data(), S.size() * 4, cudaMemcpyHostToDevice));
      if (c.dl_floats) CU(cudaMemset(c.d_dline, 0, (size_t)c.dl_floats * V * sizeof(float)));
      if (c.ring_floats) CU(cudaMemset(c.d_ring, 0, (size_t)c.ring_floats * V * sizeof(float)));
      if (c.conv) {
        CU(cudaMemset(c.d_cx, 0, (size_t)V * c.conv_stride * sizeof(float))); CU(cudaMemset(c.d_cxl, 0, (size_t)V * c.conv_stride * sizeof(float)));
        CU(launch_conv_toeplitz(reinterpret_cast<const float*>(c.d_uniform + c.conv_off + 2), c.conv_K, c.d_th, c.d_tl, c.conv_J, stream));
        CU(cudaStreamSynchronize(stream));
      }
    }
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
      std::string e = dev_alloc(&d_wtdata[kind], t.data.size());
      if (!e.empty()) return e;
      CU(cudaMemcpy(d_wtdata[kind], t.data.data(), t.data.size() * 4, cudaMemcpyHostToDevice));
      h_wt[kind].data = d_wtdata[kind];
      changed = true;
    }
    if (!d_wt) {
      std::string e = dev_alloc(&d_wt, 6);
      if (!e.empty()) return e;
      changed = true;
    }
    if (changed) CU(cudaMemcpy(d_wt, h_wt, sizeof(h_wt), cudaMemcpyHostToDevice));
  }
  if (upload_state) dirty = false;
  return "";
}

std::string Bank::set_sample_rate(double s) {  // AudioUnit::set_sample_rate
  sr = s;
  const double unit_rate = net_rate ? (double)(float)s : s;
  for (auto& n : nodes) {   // the bank of a sequencer is re-rated like the sequencer: its events' units are reset (a unit pushed later is not)
    const bool reset = event_rerate_resets(n.get(), unit_rate);
    n->set_sample_rate(unit_rate);
    if (reset) n->reset();
  }
  // Parameters always follow the new rate. State is re-initialised only while nothing has been rendered
  // (or when delay lengths change, which resets the lines like src/delay.rs:105-113).
  return lower_and_upload(!dirty);
}

std::string Bank::set(uint32_t voice, const Setting& st) {  // AudioUnit::set (src/audiounit.rs:62, src/setting.rs) on a live bank
  if (voice >= V()) return "#A set: voice index out of range";
  CU(cudaSetDevice(device));
  { std::string re = rt_stop(); if (!re.empty()) return re; } process_streak = 0;
  // the setting is tried on a COPY of the voice's host graph: a refused setting (one that would change a class-uniform word) leaves
  // both the host graph and the device untouched; the copy replaces the original only after the upload
  std::unique_ptr<HNode> trial(nodes[voice]->clone());
  trial->set(st);
  Lowering l;
  trial->lower(l);
  if (!l.ok) return "#U " + l.why;
  for (auto& c : classes) {
    auto it = std::lower_bound(c.voices.begin(), c.voices.end(), voice);
    if (it == c.voices.end() || *it != voice) continue;
    const uint32_t i = (uint32_t)(it - c.voices.begin()), Vc = c.V();
    if (l.U != c.uniform || l.P.size() != c.np || l.S.size() != c.ns)
      return "#U set: the setting changes a class-uniform word (a delay length); rebuild the bank instead";
    // parameters take effect at once (one strided column of the [NP][V] block); running state is left alone, the
    // construction-time state (what reset() restores) follows the setting like the reference's stored phase/seed
    if (c.np) CU(cudaMemcpy2DAsync(c.d_params + i, (size_t)Vc * 4, l.P.data(), 4, 4, c.np, cudaMemcpyHostToDevice, stream));
    CU(cudaStreamSynchronize(stream));  // `l` is pageable and goes out of scope
    const std::vector<uint32_t> S0 = l.reset_image();
    for (uint32_t k = 0; k < c.ns; k++) c.state0[(size_t)k * Vc + i] = S0[k];
    c.state0_stale = true;
    nodes[voice] = std::move(trial);
    return "";
  }
  return "internal: voice not found in any class";
}

double Bank::loop_point() const {
  if (!(loop_arg > 0.0)) return std::numeric_limits<double>::infinity();
  const double unit_rate = net_rate ? (double)(float)sr : sr;
  return std::max(64.0 * (1.0 / unit_rate), std::round(loop_arg * unit_rate) / unit_rate);
}
void Bank::advance_clock(uint64_t n) {   // what every Event<X> voice does to its own clock (nodes.cuh Event::plan / at_sample)
  const double unit_rate = net_rate ? (double)(float)sr : sr, sd = 1.0 / unit_rate, lp = loop_point();
  for (uint64_t t0 = 0; t0 < n; t0 += 64) {
    const uint64_t size = std::min<uint64_t>(64, n - t0);
    if (!(loop_arg > 0.0)) { seq_time = seq_time + sd * (double)size; continue; }
    const double x = std::round(std::max(0.0, lp - seq_time) * unit_rate);
    const uint64_t loop_size = x > 0.0 ? (uint64_t)x : 0;
    seq_time = std::min(seq_time + sd * (double)size, lp);
    if (loop_size < size) seq_time = std::min(0.0 + sd * (double)(size - loop_size), lp);   // wrapped: the rest of the block counts from 0
  }
}
std::string Bank::state0_to_device(VoiceClass& c, const uint32_t** out) {
  *out = nullptr;
  if (!(loop_arg > 0.0) || c.state0.empty() || c.sig.compare(0, 6, "Event<") != 0) return "";
  if (!c.d_state0) { std::string e = dev_alloc(&c.d_state0, c.state0.size()); if (!e.empty()) return e; c.state0_stale = true; }
  if (c.state0_stale) { CU(cudaMemcpy(c.d_state0, c.state0.data(), c.state0.size() * 4, cudaMemcpyHostToDevice)); c.state0_stale = false; }
  *out = c.d_state0;
  return "";
}

// `l`: the words to run with. `reset_state`: the construction-time state that reset() restores (defaults to l.S).
std::string Bank::upload_voice(uint32_t voice, const Lowering& l, bool with_state, const std::vector<uint32_t>* reset_state) {
  { std::string re = rt_stop(); if (!re.empty()) return re; } process_streak = 0;
  for (auto& c : classes) {
    auto it = std::lower_bound(c.voices.begin(), c.voices.end(), voice);
    if (it == c.voices.end() || *it != voice) continue;
    const uint32_t i = (uint32_t)(it - c.voices.begin()), Vc = c.V();
    if (l.U != c.uniform || l.P.size() != c.np || l.S.size() != c.ns || (reset_state && reset_state->size() != c.ns))
      return "#U the voice does not fit its class: a class-uniform word (delay length, table, wave) or the word layout differs; rebuild the bank instead";
    if (with_state && c.fdn) return "#U voices of a two-stage (FDN reverb) class cannot be replaced in place";
    if (c.np) CU(cudaMemcpy2DAsync(c.d_params + i, (size_t)Vc * 4, l.P.data(), 4, 4, c.np, cudaMemcpyHostToDevice, stream));
    const std::vector<uint32_t> S0 = reset_state ? *reset_state : l.reset_image();
    for (uint32_t k = 0; k < c.ns; k++) c.state0[(size_t)k * Vc + i] = S0[k];
    c.state0_stale = true;
    if (with_state) {
      if (c.ns) CU(cudaMemcpy2DAsync(c.d_state + i, (size_t)Vc * 4, l.S.data(), 4, 4, c.ns, cudaMemcpyHostToDevice, stream));
      if (c.dl_floats) CU(cudaMemset2DAsync(c.d_dline + i, (size_t)Vc * 4, 0, 4, (size_t)c.dl_floats, stream));
    }
    CU(cudaStreamSynchronize(stream));  // `l` is pageable
    return "";
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
  const double unit_rate = net_rate ? (double)(float)sr : sr;
  n->set_sample_rate(unit_rate);
  Lowering l0, l;
  n->lower(l0);                                        // what reset() restores: the event's clock at 0, like every other voice
  const bool ev = event_set_clock(n.get(), seq_time);  // an event put into a running sequencer counts from now
  n->lower(l);
  if (ev) event_set_clock(n.get(), 0.0);
  if (!l.ok) return "#U " + l.why;
  const std::vector<uint32_t> S0 = l0.reset_image();
  std::string e = upload_voice(voice, l, true, &S0);
  if (!e.empty()) return e;
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
  for (auto& c : classes) if (c.fdn || c.conv) return std::string("#U ") + what + ": banks with a two-stage class (FDN reverb, tensor-core convolver) cannot be regrouped in place; rebuild the bank";
  CU(cudaSetDevice(device));
  { std::string re = rt_stop(); if (!re.empty()) return re; } process_streak = 0;
  const double unit_rate = net_rate ? (double)(float)sr : sr;
  n->set_sample_rate(unit_rate);
  Lowering l0, l;
  n->lower(l0);                                      // (a crossfading vertex lowers as ARRIVED: a bank reset leaves it at its second unit)
  const bool xf = xfade_set_done(n.get(), false);   // ... and starts its life fading
  const bool ev = event_set_clock(n.get(), seq_time);
  n->lower(l);
  if (ev) event_set_clock(n.get(), 0.0);
  if (xf) xfade_set_done(n.get(), true);
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
      if (v == nv) {   // the newcomer: live state (an event's clock = now); what reset() restores is its construction-time state
        const std::vector<uint32_t> S0 = l0.reset_image();
        for (uint32_t k = 0; k < c.ns && k < l.S.size(); k++) { S[(size_t)k * Vc + i] = l.S[k]; c.state0[(size_t)k * Vc + i] = S0[k]; }
        c.state0_stale = true;
        if (carry) {   // a unit that keeps RUNNING inside the newcomer (the fading-out side of a crossfade): its words and delay lines move over
          for (auto& sv : saved) {
            auto it = std::lower_bound(sv.voices.begin(), sv.voices.end(), v);
            if (it == sv.voices.end() || *it != v) continue;
            const uint32_t j = (uint32_t)(it - sv.voices.begin()), Vo = (uint32_t)sv.voices.size();
            if (carry->src_s + carry->ns > sv.ns || carry->dst_s + carry->ns > c.ns || carry->src_d + carry->nd > sv.dl || carry->dst_d + carry->nd > c.dl_floats) return "internal: crossfade carry out of range";
            for (uint32_t k = 0; k < carry->ns; k++) S[(size_t)(carry->dst_s + k) * Vc + i] = sv.S[(size_t)(carry->src_s + k) * Vo + j];
            for (uint64_t q = 0; q < carry->nd; q++) D[(size_t)(carry->dst_d + q) * Vc + i] = sv.D[(size_t)(carry->src_d + q) * Vo + j];
            break;
          }
        }
        continue;
      }
      for (auto& sv : saved) {
        auto it = std::lower_bound(sv.voices.begin(), sv.voices.end(), v);
        if (it == sv.voices.end() || *it != v) continue;
        if (sv.sig != c.sig || sv.ns != c.ns || sv.dl != c.dl_floats) return "internal: a voice changed class while the bank grew";
        const uint32_t j = (uint32_t)(it - sv.voices.begin()), Vo = (uint32_t)sv.voices.size();
        for (uint32_t k = 0; k < c.ns; k++) S[(size_t)k * Vc + i] = sv.S[(size_t)k * Vo + j];
        for (uint64_t q = 0; q < c.dl_floats; q++) D[(size_t)q * Vc + i] = sv.D[(size_t)q * Vo + j];
        break;
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
  { std::string re = rt_stop(); if (!re.empty()) return re; } process_streak = 0;
  const HNode* cur = nodes[voice].get();
  Carry carry{0, 0, 0, 0, 0, 0};
  auto count = [](const HNode* h, uint32_t* ns, uint64_t* nd) { Lowering q; h->lower(q); *ns = (uint32_t)q.S.size(); *nd = 0; for (uint32_t d : q.dlen) *nd += d; return q.ok; };
  std::unique_ptr<HNode> old;
  if (const HNode* y = xfade_unit(cur, 1)) {   // the vertex crossfaded before: it must have arrived at its second unit
    for (auto& c : classes) {
      auto it = std::lower_bound(c.voices.begin(), c.voices.end(), voice);
      if (it == c.voices.end() || *it != voice) continue;
      CU(cudaStreamSynchronize(stream));
      uint32_t done = 0;
      CU(cudaMemcpy(&done, c.d_state + (size_t)(it - c.voices.begin()), 4, cudaMemcpyDeviceToHost));   // state word 0 of Xfade: done
      if (!done) {
        // Vertex::enqueue with `next` occupied: the edit waits as `latest`, a newer one replaces it (src/vertex.rs:203-218). Its program — the
        // class Xfade<second unit, new unit> the voice will move to — is compiled now, so that a unit without a device program is refused here
        std::unique_ptr<HNode> probe(mk_xfade(y->clone(), n->clone(), ease, fade_time));
        std::string sg, jerr;
        if (!probe) return "#A crossfade: the units do not fit one vertex";
        probe->set_sample_rate(net_rate ? (double)(float)sr : sr);
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
  { std::string re = rt_stop(); if (!re.empty()) return re; } process_streak = 0;
  for (auto& c : classes) {
    auto it = std::lower_bound(c.voices.begin(), c.voices.end(), voice);
    if (it == c.voices.end() || *it != voice) continue;
    const uint32_t i = (uint32_t)(it - c.voices.begin()), Vc = c.V();
    if (c.fdn || c.ns < 4 || ((c.ns - 4) & 1u) || (c.dl_floats & 1u)) return "slot: unexpected class layout";
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
    return "";
  }
  return "internal: voice not found in any class";
}

// Before a launch of n samples: a parked unit whose fade has ended is armed now (it starts fading with this launch's first block, the block
// after the one in which `next_phase` ran, src/slot.rs:163-172, src/vertex.rs:124-136); for the fades that are still running, the block in
// which each ends is found by replaying the device's per-block arithmetic (nodes.cuh Slot<X>::step in f64, Xfade<X, Y>::step in f32:
// phase_left, n_f, fade_phase += n_f / (fade_time sr)) from the voice's fade_phase word.
std::string Bank::slot_service(uint64_t n, uint64_t* cut) {
  *cut = n;
  auto locate = [&](uint32_t voice, VoiceClass** pc, uint32_t* pi) {
    for (auto& c : classes) {
      auto vi = std::lower_bound(c.voices.begin(), c.voices.end(), voice);
      if (vi != c.voices.end() && *vi == voice) { *pc = &c; *pi = (uint32_t)(vi - c.voices.begin()); return true; }
    }
    return false;
  };
  // 1. arm what is ready. Arming a vertex regroups the classes, so the scan starts over after every arm.
  for (bool again = true; again;) {
    again = false;
    CU(cudaStreamSynchronize(stream));
    for (auto it = slot_latest.begin(); it != slot_latest.end(); ++it) {
      VoiceClass* c = nullptr; uint32_t i = 0;
      if (!locate(it->first, &c, &i) || !is_slot(nodes[it->first].get())) { slot_latest.erase(it); again = true; break; }
      uint32_t has_next = 0;
      CU(cudaMemcpy(&has_next, c->d_state + (size_t)1 * c->V() + i, 4, cudaMemcpyDeviceToHost));
      if (has_next) continue;
      const uint32_t voice = it->first;
      SlotLatest w = std::move(it->second);
      slot_latest.erase(it);
      std::string e = slot_arm_now(voice, w.ease, w.fade_time, w.unit.release(), false);
      if (!e.empty()) return e;
      again = true; break;
    }
    if (again) continue;
    for (auto it = xfade_latest.begin(); it != xfade_latest.end(); ++it) {
      VoiceClass* c = nullptr; uint32_t i = 0;
      if (!locate(it->first, &c, &i) || !xfade_unit(nodes[it->first].get(), 1)) { xfade_latest.erase(it); again = true; break; }
      uint32_t done = 0;
      CU(cudaMemcpy(&done, c->d_state + i, 4, cudaMemcpyDeviceToHost));
      if (!done) continue;
      const uint32_t voice = it->first;
      SlotLatest w = std::move(it->second);
      xfade_latest.erase(it);
      std::string e = crossfade_voice(voice, w.ease, (float)w.fade_time, w.unit.release());
      if (!e.empty()) return e;
      again = true; break;
    }
  }
  // 2. where do the running fades with a parked unit end?
  auto consider = [&](uint64_t t_end) { if (t_end < *cut) *cut = t_end; };
  for (auto& kv : slot_latest) {
    VoiceClass* c = nullptr; uint32_t i = 0;
    if (!locate(kv.first, &c, &i)) continue;
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
    VoiceClass* c = nullptr; uint32_t i = 0;
    if (!locate(kv.first, &c, &i)) continue;
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
  const double unit_rate = net_rate ? (double)(float)sr : sr, sd = 1.0 / unit_rate;
  n->set_sample_rate(unit_rate);
  std::string want; n->sig(want);
  Lowering l0, l;
  n->lower(l0);                             // what reset() restores: the event's clock at 0 (ReplayMode::All replays it from the top)
  event_set_clock(n.get(), seq_time);       // the event counts from now; a start time in the past makes it sound from the next block on
  n->lower(l);
  event_set_clock(n.get(), 0.0);
  if (!l.ok) return "#U " + l.why;
  for (auto& c : classes) {
    if (c.sig != want || c.uniform != l.U || c.fdn) continue;
    for (uint32_t v : c.voices) {
      if (!event_times(nodes[v].get(), &s0, &e0)) break;
      if (!(e0 <= seq_time + 0.5 * sd)) continue;   // Event::plan's end-of-event test at the start of the next block: still sounding
      const std::vector<uint32_t> S0 = l0.reset_image();
      std::string e = upload_voice(v, l, true, &S0);
      if (!e.empty()) return e;
      nodes[v] = std::move(n);
      if (voice) *voice = v;
      return "";
    }
  }
  return "#N no finished event of the same graph class is free: create the bank with spare events of this class (finished, or ending at time 0), or rebuild it";
}

std::string Bank::reset() {  // AudioUnit::reset: back to the construction-time state
  CU(cudaSetDevice(device));
  { std::string re = rt_stop(); if (!re.empty()) return re; } process_streak = 0;
  while (!slot_latest.empty()) {   // SlotBackend::reset adopts the LATEST configuration (src/slot.rs:156-172): arm it (its words become the voice's reset image)
    auto it = slot_latest.begin();
    const uint32_t voice = it->first;
    SlotLatest w = std::move(it->second);
    slot_latest.erase(it);
    std::string e = slot_arm_now(voice, w.ease, w.fade_time, w.unit.release(), true);
    if (!e.empty()) return e;
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
    if (c.ring_floats) CU(cudaMemsetAsync(c.d_ring, 0, (size_t)c.ring_floats * c.V() * sizeof(float), stream));
    if (c.conv) { CU(cudaMemsetAsync(c.d_cx, 0, (size_t)c.V() * c.conv_stride * sizeof(float), stream)); CU(cudaMemsetAsync(c.d_cxl, 0, (size_t)c.V() * c.conv_stride * sizeof(float), stream)); }
  }
  CU(cudaStreamSynchronize(stream));
  dirty = false; seq_time = 0.0;
  return "";
}

// long launches of wavetable programs stage the table set in shared memory (TMA bulk copy, ~160 KB per CTA); short ones
// (process()-sized) read the tables through L1/L2 instead
static size_t table_bytes_of(const VoiceClass& c, uint32_t len) {
  const int wk = c.k ? c.k->wave_kind : -1;
  static const uint32_t tb_min = [] { const char* e = getenv("FDSP_TB_MIN"); return e ? (uint32_t)atoi(e) : 32u; }();  // at 64 samples the TMA-staged tables already win
  return (wk >= 0 && len >= tb_min) ? device_wavetable(wk).data.size() * sizeof(float) : 0;
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
// FDSP_STAGED=0 switches them off (A/B), FDSP_STAGED_MAXV moves the class-size bound.
static bool use_staged(const Program* k, uint32_t V, uint32_t len, uint32_t sms) {
  const char* e = getenv("FDSP_STAGED");            // read per call: the tests toggle it inside one process
  const char* m = getenv("FDSP_STAGED_MAXV");
  const int on = e ? atoi(e) : 1;
  const uint32_t maxv = m ? (uint32_t)atoi(m) : sms * 32u;
  return on != 0 && k && k->stages >= 2 && len >= 256u && V <= maxv;
}
// CTA shape of a stage-pipelined class: 32 voices per CTA while that still leaves SMs free, else 128 with the voices spread evenly
// (FDSP_STAGED_W=128 forces the wide shape: lets the tests reach it with few voices)
static uint32_t staged_grid(uint32_t V, uint32_t sms, uint32_t* vpc) {
  const char* w = getenv("FDSP_STAGED_W");
  if (V <= sms * 32u && !(w && atoi(w) == 128)) { *vpc = 32u; return (V + 31u) / 32u; }
  return bank_grid(V, 128u, sms, vpc);
}

// ---- resident process() kernel
// A resident kernel holds a CTA (and, with staged wavetables, nearly all shared memory) on every SM: anything else launched on the device
// would sit behind it until its idle time-out. So at most one bank per device keeps one, and every entry point of EVERY bank of that
// device — they all begin with rt_stop() — first asks the owner to leave. (Banks of one device are driven from one thread at a time,
// like the units of the reference's audio thread; the registry itself is locked.)
std::string Bank::rt_stop() {
  Bank* other = nullptr;
  if (device >= 0 && device < 64) { std::lock_guard<std::mutex> lock(g_rt_mu); other = g_rt_owner[device]; if (other == this || (other && !other->rt_running)) other = nullptr; }
  if (other) { std::string e = other->rt_stop(); if (!e.empty()) return e; }
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
  if (c.fdn || c.conv || !c.k || !c.k->has_rt) return "";
  uint32_t vpc = (uint32_t)c.k->threads;
  const uint32_t grid = bank_grid(c.V(), (uint32_t)c.k->threads, sm_count(device), &vpc);
  if (grid > sm_count(device)) return "";           // every CTA must be resident at once
  if (++process_streak < 3u && !rt_running) return "";   // a bank that is driven block by block: the third process() call in a row starts the kernel
  if (!rt_running) { std::string re = rt_stop(); if (!re.empty()) return re; }   // (another bank of this device may own the resident slot)
  if (!rt_ctl) {
    CU(cudaHostAlloc((void**)&rt_ctl, sizeof(RtCtl), cudaHostAllocMapped));
    CU(cudaHostGetDevicePointer((void**)&rt_ctl_dev, rt_ctl, 0));
    CU(cudaMalloc((void**)&d_rt_relay, 16));
  }
  if (rt_partial_cap < (size_t)grid * nout * 64) { cudaFree(d_rt_partial); d_rt_partial = nullptr; CU(cudaMalloc((void**)&d_rt_partial, (size_t)grid * nout * 64 * 4)); rt_partial_cap = (size_t)grid * nout * 64; }
  if (!rt_running) {
    const uint32_t first = ++rt_seq; if (rt_seq >= 0xfffffff0u) rt_seq = 1;
    memset((void*)rt_ctl, 0, sizeof(RtCtl));
    rt_ctl->doorbell = first - 1u; rt_ctl->done = first - 1u;
    const uint32_t relay[4] = {first - 1u, 0u, 0u, 0u};
    CU(cudaMemcpyAsync(d_rt_relay, relay, 16, cudaMemcpyHostToDevice, stream));
    CU(cudaMemsetAsync(d_ticket, 0, 4, stream));
    BankArgs a;
    { std::string se = state0_to_device(c, &a.state0); if (!se.empty()) return se; } a.dl_floats = (uint32_t)c.dl_floats;
    a.params = c.d_params; a.state = c.d_state; a.uniform = c.d_uniform; a.dline = c.d_dline; a.wt = d_wt; a.in = nullptr; a.out = nullptr; a.partial = d_rt_partial;
    a.V = c.V(); a.n = 64; a.vpc = vpc; a.in_stride = 0; a.in_offset = 0; a.out_stride = 0; a.out_offset = 0; a.row_map = c.d_rowmap;
    a.sr = (float)sr; a.sd64 = (float)(1.0 / sr); a.sd32 = 1.0f / (float)sr; a.ticket = d_ticket; a.mix = nullptr; a.mix_stride = 0; a.mix_offset = 0; a.mix_accumulate = 0;
    RtArgs rt{rt_ctl_dev, d_rt_relay, first};
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
  if (dom_n == dom_ev.size()) { cudaEvent_t e; CU(cudaEventCreate(&e)); dom_ev.push_back(e); }
  CU(cudaEventRecord(dom_ev[dom_n++], st));
  return "";
}

std::string Bank::render_device(uint64_t n, const float* in_dev, uint64_t in_stride, float* out_dev, uint64_t out_stride, float* mix_dev,
                                uint64_t mix_stride) {
  if (!has_parked()) return render_device_run(n, in_dev, in_stride, out_dev, out_stride, mix_dev, mix_stride);
  // parked Slot updates: the launch is cut behind the block in which a running fade ends, the parked unit is armed, the rest follows
  CU(cudaSetDevice(device));
  { std::string re = rt_stop(); if (!re.empty()) return re; }
  uint64_t done = 0;
  do {
    uint64_t cut = n - done;
    std::string e = slot_service(n - done, &cut);
    if (!e.empty()) return e;
    if (cut == 0) break;
    e = render_device_run(cut, in_dev ? in_dev + done : nullptr, in_stride, out_dev ? out_dev + done : nullptr, out_stride, mix_dev ? mix_dev + done : nullptr, mix_stride);
    if (!e.empty()) return e;
    done += cut;
  } while (done < n);
  return "";
}

std::string Bank::render_device_run(uint64_t n, const float* in_dev, uint64_t in_stride, float* out_dev, uint64_t out_stride, float* mix_dev,
                                    uint64_t mix_stride) {
  CU(cudaSetDevice(device));
  { std::string re = rt_stop(); if (!re.empty()) return re; }
  if (!in_process) process_streak = 0;
  if (nin > 0 && !in_dev) return "#A bank has inputs but no input buffer was given";
  const bool want_v = (out_mode & 1u) && out_dev, want_m = (out_mode & 2u) && mix_dev;
  if (!want_v && !want_m) return "#A no output buffer matches the bank's out_mode";
  if (n == 0) return "";
  const bool save_want_m_ = want_m;
  if (in_stride > 0xffffffffull || out_stride > 0xffffffffull || mix_stride > 0xffffffffull) return "#A stride too large";
  if (timing) { CU(cudaEventRecord(ev0, stream)); dom_n = 0; }
  // Net-ordered mix: the voice kernels materialise per-voice rows (user buffer, or an internal one) and tree_mix_kernel adds
  // them in the Net's association order; the CTA-level partial mix is bypassed.
  const bool tree = tree_mix != 0 && want_m;
  // two-stage classes (fused dry program + warp-per-voice FDN) run as a two-stream software pipeline over PIPE_CHUNK samples
  bool pipelined = false;
  if (!tree && !getenv("FDSP_NO_PIPELINE")) for (auto& c : classes) pipelined = pipelined || (c.fdn && c.k);
  const uint32_t CH = tree ? 4096u : (pipelined ? PIPE_CHUNK : TIME_CHUNK);
  struct Pending { VoiceClass* c; uint32_t grid, len; uint64_t t0; int buf; };
  std::vector<Pending> pending;   // deferred CTA-partial reductions of pipelined classes (issued one chunk late, on `stream`)
  auto flush_pending = [&](VoiceClass* only) -> std::string {
    for (size_t q = 0; q < pending.size();) {
      Pending& pd = pending[q];
      if (only && pd.c != only) { q++; continue; }
      CU(cudaStreamWaitEvent(stream, pd.c->e_fdn[pd.buf], 0));
      if (save_want_m_) { CU(launch_mix_reduce(pd.buf ? pd.c->d_partial2 : pd.c->d_partial, pd.grid, (uint32_t)nout, pd.len, mix_dev, (uint32_t)mix_stride, (uint32_t)pd.t0, 1, stream)); launches++; }
      pending.erase(pending.begin() + (long)q);
    }
    return "";
  };
  uint64_t chunk_index = 0;
  bool joined = true;
  // FDSP_PIPE_TRACE=1: print the device timeline of the two pipeline stages (diagnostic; synchronises)
  const bool trace = pipelined && getenv("FDSP_PIPE_TRACE") != nullptr;
  std::vector<cudaEvent_t> tev;   // per chunk: dry start, dry end, fdn start, fdn end
  auto tmark = [&](cudaStream_t st) { if (trace) { cudaEvent_t e; cudaEventCreate(&e); cudaEventRecord(e, st); tev.push_back(e); } };
  if (tree && !want_v) {
    const size_t need = (size_t)V() * nout * CH;
    if (rows_cap < need) { std::string e = dev_alloc(&d_rows, need); if (!e.empty()) return e; rows_cap = need; }
  }
  const bool save_want_v = want_v, save_want_m = want_m;
  // pipelined banks accumulate into a zeroed mix: cleared once for the whole call, so that nothing sits between the dry-stage launches of
  // consecutive chunks on `stream` (a gap there lets the wide FDN kernel of the previous chunk take every SM first)
  if (pipelined && save_want_m) CU(cudaMemset2DAsync(mix_dev, (size_t)mix_stride * 4, 0, (size_t)n * 4, (size_t)nout, stream));
  for (uint64_t t0 = 0; t0 < n; t0 += CH, chunk_index++) {
    const uint32_t len = (uint32_t)std::min<uint64_t>(CH, n - t0);
    bool first = true;
    if (pipelined && save_want_m) first = false;   // every class accumulates into the mix region zeroed above (reductions of pipelined classes arrive late)
    bool want_v = save_want_v, want_m = save_want_m;
    float* out_dev_c = out_dev; uint64_t out_stride_c = out_stride; uint64_t out_t0 = t0;
    if (tree) { want_m = false; if (!save_want_v) { want_v = true; out_dev_c = d_rows; out_stride_c = CH; out_t0 = 0; } }
    const int mode = (want_v ? 1 : 0) | (want_m ? 2 : 0);
    // several plain classes: launch the class kernels concurrently (own streams, forked from and joined back into `stream`); the
    // partial mixes are still reduced on `stream` in class order, so the result does not depend on how the kernels overlap
    bool concurrent = classes.size() > 1 && !pipelined && len > 64 && !getenv("FDSP_NO_CONCURRENT");
    for (auto& c : classes) concurrent = concurrent && !c.fdn;
    if (concurrent) CU(cudaEventRecord(e_begin, stream));
    // (Launching the class with the longest dependency chain first, on a high-priority stream, is worse for config 5 than class order:
    // its CTAs hold ~195 KB of shared memory, so every light class then waits for all of it.
    // FDSP_HEAVY_FIRST=1 keeps that order for experiments; FDSP_CARVEOUT=<percent> makes every class kernel ask for the same carve-out.)
    std::vector<size_t> order(classes.size());
    for (size_t q = 0; q < order.size(); q++) order[q] = q;
    if (concurrent && getenv("FDSP_HEAVY_FIRST"))
      std::stable_sort(order.begin(), order.end(), [&](size_t x, size_t y) { return (classes[x].k && classes[x].k->stages > 1) > (classes[y].k && classes[y].k->stages > 1); });
    struct CarveGuard { int saved; CarveGuard() : saved(launch_carveout()) {} ~CarveGuard() { launch_carveout() = saved; } } carve_guard;
    // Concurrent classes ask for ONE carve-out, the maximum: the class that stages the wavetables (~195 KB per CTA) needs it anyway, and kernels
    // that prefer different L1 / shared-memory splits do not share an SM.
    if (concurrent) { const char* cv = getenv("FDSP_CARVEOUT"); launch_carveout() = cv ? atoi(cv) : 100; }
    for (size_t oi = 0; oi < order.size(); oi++) {
      auto& c = classes[order[oi]];
      const uint32_t V = c.V();
      cudaStream_t ks = stream;
      if (concurrent) {
        if (!c.cstream) { CU(cudaStreamCreateWithFlags(&c.cstream, cudaStreamNonBlocking)); CU(cudaEventCreateWithFlags(&c.e_done, cudaEventDisableTiming)); }
        ks = c.cstream;
        CU(cudaStreamWaitEvent(ks, e_begin, 0));
      }
      const uint32_t nsm = sm_count(device);
      const bool staged = use_staged(c.k.get(), V, len, nsm);
      int fdn_warps = 1;   // voices (= warps) per CTA of the FDN kernel
      if (c.fdn) {
        const int cap = fdn_max_warps();
        // pipelined: leave SMs free for the CTAs of the dry stage of the next chunk (their shared-memory tables cannot share an SM
        // with an FDN CTA), otherwise the two stages serialise on SM residency
        uint32_t sms = nsm;
        if (pipelined && c.k) { uint32_t dv = 0; const uint32_t dry_ctas = staged ? staged_grid(V, nsm, &dv) : (V + (uint32_t)c.k->threads - 1) / (uint32_t)c.k->threads; sms = dry_ctas < nsm / 2 ? nsm - dry_ctas : nsm / 2; }
        fdn_warps = (int)((V + sms - 1) / sms); if (fdn_warps > cap) fdn_warps = cap; if (fdn_warps < 1) fdn_warps = 1;
      }
      // voice programs: whole waves of CTAs with the voices spread evenly; the dry stage of a two-stage class stays compact
      // (few CTAs) so that it leaves the other SMs to the FDN kernel it is pipelined with
      uint32_t vpc = c.k ? (uint32_t)c.k->threads : 0u;
      const uint32_t vgrid = !c.k ? 0u : (staged ? staged_grid(V, nsm, &vpc) : (c.fdn || getenv("FDSP_NO_SPREAD") ? (V + vpc - 1) / vpc : bank_grid(V, (uint32_t)c.k->threads, nsm, &vpc)));
      auto launch_voice = [&](const BankArgs& args, int md, cudaStream_t st) { return staged ? c.k->launch_staged(args, md, table_bytes_of(c, len), st) : c.k->launch(args, md, table_bytes_of(c, len), st); };
      const uint32_t grid = c.fdn ? V : vgrid;   // rows of the partial-mix buffer: one per CTA of a voice program, one per VOICE of the FDN kernel (its warps never meet)
      if (c.conv) {
        // stage 1: the program in front of the convolver writes its rows behind the history columns; then x_lo, the Toeplitz GEMM tiles
        // (rows straight into the caller's buffer, or an internal one), the history shift, and the voice-order fold of the rows
        BankArgs d{};
        d.params = c.d_params; d.state = c.d_state; d.uniform = c.d_uniform; d.dline = c.d_dline; d.wt = d_wt; d.in = in_dev; d.partial = nullptr;
        d.out = c.d_cx; d.V = V; d.n = len; d.vpc = vpc; d.in_stride = (uint32_t)in_stride; d.in_offset = (uint32_t)t0; d.out_stride = c.conv_stride; d.out_offset = c.conv_H;
        d.row_map = c.d_dryrows; d.sr = (float)sr; d.sd64 = (float)(1.0 / sr); d.sd32 = 1.0f / (float)sr; d.ticket = nullptr; d.mix = nullptr; d.mix_stride = 0; d.mix_offset = 0; d.mix_accumulate = 0;
        CU(launch_voice(d, 1, stream));
        CU(launch_conv_split(c.d_cx, c.d_cxl, V, c.conv_stride, c.conv_H, len, stream));
        float* y = want_v ? out_dev_c : nullptr; uint32_t ys = (uint32_t)out_stride_c, yo = (uint32_t)out_t0;
        if (!y) {
          if (c.crows_cap < (size_t)V * TIME_CHUNK) { std::string e = dev_alloc(&c.d_crows, (size_t)V * TIME_CHUNK); if (!e.empty()) return e; c.crows_cap = (size_t)V * TIME_CHUNK; }
          y = c.d_crows; ys = TIME_CHUNK; yo = 0;
        }
        { std::string de = dom_mark(stream); if (!de.empty()) return de; }
        CU(launch_conv_tc(c.conv_maps, y, ys, yo, c.d_dryrows, V, len, c.conv_K, c.conv_H, stream));
        { std::string de = dom_mark(stream); if (!de.empty()) return de; }
        CU(launch_conv_history(c.d_cx, c.d_cxl, V, c.conv_stride, c.conv_H, len, stream));
        launches += 4;
        if (want_m) { CU(launch_tree_mix(y, V, 1u, ys, yo, len, mix_dev, (uint32_t)mix_stride, (uint32_t)t0, 0, stream)); launches++; }
        first = false;
        continue;
      }
      if (want_m) {
        const size_t need = (size_t)grid * nout * len;
        if (c.partial_floats < need) { std::string e = dev_alloc(&c.d_partial, (size_t)grid * nout * TIME_CHUNK); if (!e.empty()) return e; c.partial_floats = (size_t)grid * nout * TIME_CHUNK; }
        if (pipelined && c.fdn && c.k && c.partial2_floats < need) { std::string e = dev_alloc(&c.d_partial2, (size_t)grid * nout * PIPE_CHUNK); if (!e.empty()) return e; c.partial2_floats = (size_t)grid * nout * PIPE_CHUNK; }
      }
      BankArgs a;
      { std::string se = state0_to_device(c, &a.state0); if (!se.empty()) return se; } a.dl_floats = (uint32_t)c.dl_floats;
      a.params = c.d_params; a.state = c.d_state; a.uniform = c.d_uniform; a.dline = c.d_dline; a.wt = d_wt;
      a.in = in_dev; a.out = want_v ? out_dev_c : nullptr; a.partial = want_m ? c.d_partial : nullptr;
      a.V = V; a.n = len; a.vpc = vpc;
      a.in_stride = (uint32_t)in_stride; a.in_offset = (uint32_t)t0;
      a.out_stride = (uint32_t)out_stride_c; a.out_offset = (uint32_t)out_t0;
      a.row_map = c.d_rowmap;
      a.sr = (float)sr; a.sd64 = (float)(1.0 / sr); a.sd32 = 1.0f / (float)sr;
      // process()-sized launches of plain voice programs finish their mix-down inside the kernel (one launch instead of two)
      const bool fused_mix = want_m && !c.fdn && len <= 64;
      a.ticket = fused_mix ? d_ticket : nullptr; a.mix = mix_dev; a.mix_stride = (uint32_t)mix_stride; a.mix_offset = (uint32_t)t0; a.mix_accumulate = first ? 0 : 1;
      if (t0 > 0xffffffffull - TIME_CHUNK) return "#A render too long for one call";
      if (c.fdn && len > TIME_CHUNK) return "internal: chunk";
      // long launches of wavetable programs stage the table set in shared memory (TMA bulk copy, ~160 KB per CTA);
      // short ones (process()-sized) read the tables through L1/L2 instead
      if (c.fdn) {
        FdnArgs f;
        f.params = c.d_params; f.state = c.d_state; f.uniform = c.d_uniform; f.p0 = c.p0; f.s0 = c.s0; f.u0 = c.u0; f.scalar_row = c.scalar_row;
        if (c.k && pipelined) {
          // stage 1 of chunk k on `stream`, stage 2 on `stream2`; buffers alternate, chunk k-1's partial mix is reduced after
          // stage 1 of chunk k has been queued so that the two stages of neighbouring chunks run side by side
          const int buf = (int)(chunk_index & 1);
          float* dry = buf ? c.d_dry2 : c.d_dry;
          CU(cudaStreamWaitEvent(stream, c.e_fdn[buf], 0));   // FDN of chunk k-2 has consumed this dry buffer (no-op before the first record)
          BankArgs d = a;
          d.out = dry; d.partial = nullptr; d.out_stride = PIPE_CHUNK; d.out_offset = 0; d.row_map = c.d_dryrows;
          tmark(stream);
          CU(launch_voice(d, 1, stream));
          launches++;
          tmark(stream);
          CU(cudaEventRecord(c.e_dry[buf], stream));
          // A bank of this one class keeps `stream` for the dry stage alone — chunk k + 1 follows chunk k with nothing in between, so it
          // holds its SMs before the wide FDN kernel of chunk k floods the rest — and reduces on stream2 behind the FDN kernel. With other
          // classes in the bank every reduction stays on `stream` (they accumulate into the same mix region), one chunk late.
          const bool solo = classes.size() == 1;
          if (!solo) { std::string pe = flush_pending(&c); if (!pe.empty()) return pe; }   // reduce chunk k-1 of this class (waits for its FDN)
          f.dry = dry; f.dry_voice_stride = 2ull * PIPE_CHUNK; f.dry_ch_stride = PIPE_CHUNK; f.dry_offset = 0;
          f.out = want_v ? out_dev_c : nullptr; f.row_map = c.d_rowmap; f.out_stride = (uint32_t)out_stride_c; f.out_offset = (uint32_t)out_t0;
          f.partial = want_m ? (buf ? c.d_partial2 : c.d_partial) : nullptr;
          f.ring = c.d_ring; f.ring_voice_stride = c.ring_floats; f.V = V; f.n = len;
          CU(cudaStreamWaitEvent(stream2, c.e_dry[buf], 0));
          tmark(stream2);
          { std::string de = dom_mark(stream2); if (!de.empty()) return de; }
          CU(launch_fdn(f, fdn_warps, stream2));
          { std::string de = dom_mark(stream2); if (!de.empty()) return de; }
          launches++;
          tmark(stream2);
          CU(cudaEventRecord(c.e_fdn[buf], stream2));
          if (!solo) pending.push_back({&c, grid, len, t0, buf});
          else {
            if (want_m) { CU(launch_mix_reduce(buf ? c.d_partial2 : c.d_partial, grid, (uint32_t)nout, len, mix_dev, (uint32_t)mix_stride, (uint32_t)t0, 1, stream2)); launches++; }
            joined = false;   // stream2 carries work `stream` has not waited for (rows written by the FDN kernel, the reduction): joined after the loop
          }
          continue;
        }
        if (c.k) {  // stage 1: the fused dry program writes stereo rows [V][2][TIME_CHUNK]
          BankArgs d = a;
          d.out = c.d_dry; d.partial = nullptr; d.out_stride = TIME_CHUNK; d.out_offset = 0; d.row_map = c.d_dryrows;
          CU(launch_voice(d, 1, stream));
          launches++;
          f.dry = c.d_dry; f.dry_voice_stride = 2ull * TIME_CHUNK; f.dry_ch_stride = TIME_CHUNK; f.dry_offset = 0;
        } else {    // reverb applied straight to the bank's stereo input
          f.dry = in_dev; f.dry_voice_stride = 0; f.dry_ch_stride = (uint32_t)in_stride; f.dry_offset = (uint32_t)t0;
        }
        f.out = want_v ? out_dev_c : nullptr; f.row_map = c.d_rowmap; f.out_stride = (uint32_t)out_stride_c; f.out_offset = (uint32_t)out_t0;
        f.partial = want_m ? c.d_partial : nullptr;
        f.ring = c.d_ring; f.ring_voice_stride = c.ring_floats; f.V = V; f.n = len;
        { std::string de = dom_mark(stream); if (!de.empty()) return de; }
        CU(launch_fdn(f, fdn_warps, stream));
        { std::string de = dom_mark(stream); if (!de.empty()) return de; }
      } else {
        { std::string de = dom_mark(ks); if (!de.empty()) return de; }
        CU(launch_voice(a, mode, ks));
        { std::string de = dom_mark(ks); if (!de.empty()) return de; }
      }
      launches++;
      if (concurrent) { CU(cudaEventRecord(c.e_done, ks)); continue; }   // reduced below, after every class has been launched
      if (want_m && !fused_mix) {
        CU(launch_mix_reduce(c.d_partial, grid, (uint32_t)nout, len, mix_dev, (uint32_t)mix_stride, (uint32_t)t0, first ? 0 : 1, stream));
        launches++;
      }
      first = false;
    }
    if (concurrent) {
      for (auto& c : classes) {
        CU(cudaStreamWaitEvent(stream, c.e_done, 0));
        if (want_m) {
          uint32_t vpc = (uint32_t)c.k->threads;
          const uint32_t nsm = sm_count(device);
          const uint32_t grid = use_staged(c.k.get(), c.V(), len, nsm) ? staged_grid(c.V(), nsm, &vpc) : (getenv("FDSP_NO_SPREAD") ? (c.V() + vpc - 1) / vpc : bank_grid(c.V(), (uint32_t)c.k->threads, nsm, &vpc));
          CU(launch_mix_reduce(c.d_partial, grid, (uint32_t)nout, len, mix_dev, (uint32_t)mix_stride, (uint32_t)t0, first ? 0 : 1, stream));
          launches++;
        }
        first = false;
      }
    }
    if (tree) {
      const size_t sc = tree_mix == 1 ? tree_mix_scratch_floats(V(), (uint32_t)nout, CH) : 0;   // balanced tree of a big bank: subtree sums first
      if (sc > treepart_cap) { std::string e = dev_alloc(&d_treepart, sc); if (!e.empty()) return e; treepart_cap = sc; }
      CU(launch_tree_mix(out_dev_c, V(), (uint32_t)nout, (uint32_t)out_stride_c, (uint32_t)out_t0, len, mix_dev, (uint32_t)mix_stride, (uint32_t)t0, tree_mix == 1 ? 1 : 0, stream, sc ? d_treepart : nullptr));
      launches += sc ? 2 : 1;
    }
  }
  { std::string pe = flush_pending(nullptr); if (!pe.empty()) return pe; }   // also joins stream2 back into `stream`
  if (!joined) { CU(cudaEventRecord(e_begin, stream2)); CU(cudaStreamWaitEvent(stream, e_begin, 0)); }   // solo two-stage class: its reductions ran on stream2
  if (timing) CU(cudaEventRecord(ev1, stream));
  if (trace) {
    CU(cudaStreamSynchronize(stream));
    for (size_t q = 0; q + 3 < tev.size(); q += 4) {
      float t[4];
      for (int w = 0; w < 4; w++) cudaEventElapsedTime(&t[w], ev0, tev[q + w]);
      fprintf(stderr, "[pipe] chunk %zu: dry %.3f..%.3f ms   fdn %.3f..%.3f ms\n", q / 4, t[0], t[1], t[2], t[3]);
    }
    for (auto e : tev) cudaEventDestroy(e);
  }
  dirty = true; advance_clock(n);
  return "";
}

std::string Bank::ensure_staging(uint32_t chunk) {
  { std::string re = rt_stop(); if (!re.empty()) return re; }   // allocations synchronise with the device: no resident kernel may be waiting on its doorbell
  const size_t rows = (size_t)V() * nout;
  std::string e;
  if (nin > 0 && in_cap < (size_t)nin * chunk) { if (!(e = dev_alloc(&d_in, (size_t)nin * chunk)).empty()) return e; in_cap = (size_t)nin * chunk; }
  if ((out_mode & 1u) && out_cap < rows * chunk) { if (!(e = dev_alloc(&d_out, rows * chunk)).empty()) return e; out_cap = rows * chunk; }
  if ((out_mode & 2u) && mix_cap < (size_t)nout * chunk) { if (!(e = dev_alloc(&d_mix, (size_t)nout * chunk)).empty()) return e; mix_cap = (size_t)nout * chunk; }
  stage_chunk = std::max(stage_chunk, chunk);
  return "";
}

std::string Bank::render_host(uint64_t n, const float* in, float* out_voices, float* out_mix) {
  CU(cudaSetDevice(device));
  { std::string re = rt_stop(); if (!re.empty()) return re; }
  if (n == 0) return "";
  const size_t rows = (size_t)V() * nout;
  // chunk so that the per-voice staging buffer stays below ~512 MB
  uint32_t chunk = TIME_CHUNK;
  if ((out_mode & 1u) && out_voices) {
    const uint64_t cap = (512ull << 20) / (rows * 4);
    chunk = (uint32_t)std::max<uint64_t>(64, std::min<uint64_t>(TIME_CHUNK, cap / 64 * 64));
  }
  chunk = (uint32_t)std::min<uint64_t>(chunk, (n + 63) / 64 * 64);
  std::string e = ensure_staging(chunk);
  if (!e.empty()) return e;
  for (uint64_t t0 = 0; t0 < n; t0 += chunk) {
    const uint32_t len = (uint32_t)std::min<uint64_t>(chunk, n - t0);
    if (nin > 0) {
      if (!in) return "#A bank has inputs but no input buffer was given";
      CU(cudaMemcpy2DAsync(d_in, (size_t)chunk * 4, in + t0, (size_t)n * 4, (size_t)len * 4, nin, cudaMemcpyHostToDevice, stream));
    }
    e = render_device(len, d_in, chunk, (out_voices ? d_out : nullptr), chunk, (out_mix ? d_mix : nullptr), chunk);
    if (!e.empty()) return e;
    if (out_voices && (out_mode & 1u)) CU(cudaMemcpy2DAsync(out_voices + t0, (size_t)n * 4, d_out, (size_t)chunk * 4, (size_t)len * 4, rows, cudaMemcpyDeviceToHost, stream));
    if (out_mix && (out_mode & 2u)) CU(cudaMemcpy2DAsync(out_mix + t0, (size_t)n * 4, d_mix, (size_t)chunk * 4, (size_t)len * 4, nout, cudaMemcpyDeviceToHost, stream));
  }
  CU(cudaStreamSynchronize(stream));
  return "";
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
  std::string e = ensure_staging(64);
  if (!e.empty()) return e;
  const bool mix = (out_mode & 2u) != 0;  // mix mode wins for the AudioUnit surface; voices mode returns V*c channels
  const size_t rows = mix ? (size_t)nout : (size_t)V() * nout;
  if (h_in_cap < (size_t)std::max(1, nin) * 64) { if (h_in) cudaFreeHost(h_in); CU(cudaMallocHost((void**)&h_in, (size_t)std::max(1, nin) * 64 * 4)); h_in_cap = (size_t)std::max(1, nin) * 64; }
  if (h_out_cap < rows * 64) {
    if (h_out) cudaFreeHost(h_out);
    CU(cudaHostAlloc((void**)&h_out, rows * 64 * 4, cudaHostAllocMapped));   // mapped: the mix is written straight into it by the GPU
    CU(cudaHostGetDevicePointer((void**)&d_hout, h_out, 0));
    h_out_cap = rows * 64;
  }
  if (nin > 0) {
    if (!in) return "#A bank has inputs but no input buffer was given";
    memcpy(h_in, in, (size_t)nin * 64 * 4);
    CU(cudaMemcpyAsync(d_in, h_in, (size_t)nin * 64 * 4, cudaMemcpyHostToDevice, stream));
  }
  struct NoTiming { bool& t; explicit NoTiming(bool& x) : t(x) { t = false; } ~NoTiming() { t = true; } } no_timing(timing);  // no event records on this path
  struct InProcess { bool& f; explicit InProcess(bool& x) : f(x) { f = true; } ~InProcess() { f = false; } } in_proc(in_process);
  bool two_stage = false;   // pipelined classes clear / accumulate the mix region on the device: keep that in device memory
  for (auto& c : classes) two_stage = two_stage || (c.fdn && c.k);
  if (mix && two_stage) {
    e = render_device(size, d_in, 64, nullptr, 64, d_mix, 64);
    if (!e.empty()) return e;
    CU(cudaMemcpyAsync(h_out, d_mix, rows * 64 * 4, cudaMemcpyDeviceToHost, stream));
  } else if (mix) {
    // one block of mix is a few hundred bytes: mix_reduce_kernel stores it over PCIe into the mapped host buffer, which saves
    // the separate device-to-host copy of the latency-critical process() path
    e = render_device(size, d_in, 64, nullptr, 64, d_hout, 64);
    if (!e.empty()) return e;
  } else {
    e = render_device(size, d_in, 64, d_out, 64, nullptr, 64);
    if (!e.empty()) return e;
    CU(cudaMemcpyAsync(h_out, d_out, rows * 64 * 4, cudaMemcpyDeviceToHost, stream));
  }
  CU(cudaStreamSynchronize(stream));
  memcpy(out, h_out, rows * 64 * 4);
  return "";
}

std::string Bank::clone_into(Bank& dst) const {
  { std::string re = const_cast<Bank*>(this)->rt_stop(); if (!re.empty()) return re; }
  std::vector<HNode*> copies;
  for (auto& n : nodes) copies.push_back(n->clone());
  dst.sr = sr; dst.tree_mix = tree_mix; dst.net_rate = net_rate; dst.vertex_of_voice = vertex_of_voice;
  std::string e = dst.init(copies, device, out_mode);
  if (!e.empty()) return e;
  for (auto& n : dst.nodes) n->set_sample_rate(sr);
  if (!(e = dst.lower_and_upload(true)).empty()) return e;
  CU(cudaSetDevice(device));
  CU(cudaStreamSynchronize(stream));
  for (size_t i = 0; i < classes.size(); i++) {
    const VoiceClass& s = classes[i]; VoiceClass& d = dst.classes[i];
    if (!s.state0.empty()) CU(cudaMemcpy(d.d_state, s.d_state, s.state0.size() * 4, cudaMemcpyDeviceToDevice));
    if (s.dl_floats) CU(cudaMemcpy(d.d_dline, s.d_dline, (size_t)s.dl_floats * s.V() * 4, cudaMemcpyDeviceToDevice));
    if (s.ring_floats && s.d_ring && d.d_ring) CU(cudaMemcpy(d.d_ring, s.d_ring, (size_t)s.ring_floats * s.V() * 4, cudaMemcpyDeviceToDevice));
    if (s.conv && d.conv) { CU(cudaMemcpy(d.d_cx, s.d_cx, (size_t)s.V() * s.conv_stride * 4, cudaMemcpyDeviceToDevice)); CU(cudaMemcpy(d.d_cxl, s.d_cxl, (size_t)s.V() * s.conv_stride * 4, cudaMemcpyDeviceToDevice)); }
  }
  dst.dirty = dirty; dst.seq_time = seq_time;
  for (auto& kv : slot_latest) { SlotLatest& w = dst.slot_latest[kv.first]; w.unit.reset(kv.second.unit->clone()); w.ease = kv.second.ease; w.fade_time = kv.second.fade_time; }
  for (auto& kv : xfade_latest) { SlotLatest& w = dst.xfade_latest[kv.first]; w.unit.reset(kv.second.unit->clone()); w.ease = kv.second.ease; w.fade_time = kv.second.fade_time; }
  return "";
}

}  // namespace host
}  // namespace fdsp

// fundsp_b200 bank runtime: V voices of one or more structural classes resident on one GPU.
// Host mirror of "a Vec of V AudioUnits + mix" driven like Wave::render (reference src/wave.rs:441-466).
#pragma once
#include <cuda_runtime.h>

#include <map>
#include <memory>
#include <string>
#include <vector>

#include "cuda_owned.h"
#include "graph.h"
#include "registry.h"
#include "../dsp/rt_args.h"

namespace fdsp {
namespace host {

// Error convention of the runtime: "" = ok, otherwise the message, which may start with a status tag that csrc/capi.cpp turns into the
// ABI's code and strips: "#U " unsupported (FDSP_ERR_UNSUPPORTED), "#A " bad argument (FDSP_ERR_ARG), "#N " no free slot (push_event falls
// back to growing the bank). Untagged messages are device / driver failures (FDSP_ERR_CUDA). Codes never depend on the wording.
struct VoiceClass {
  std::string sig;
  std::shared_ptr<const Program> k;
  std::vector<uint32_t> voices;     // global voice indices, ascending
  std::vector<uint32_t> uniform;    // class-uniform words (delay lengths ...)
  uint64_t dl_floats = 0;           // delay-line floats per voice (thread-per-voice layout [pos][voice])
  uint32_t np = 0, ns = 0, nu = 0;  // words per voice (whole graph)
  // reverb_stereo tail handled by the warp-per-voice FDN kernel (dsp/fdn_kernel.cuh); `k` is then the dry-stage program (may be null)
  bool fdn = false; int scalar_row = -1; uint32_t p0 = 0, s0 = 0, u0 = 0; uint64_t ring_floats = 0;
  Array<float> d_ring, d_dry; Array<uint32_t> d_dryrows;
  // `... >> convolve(h)` tail on tensor cores (dsp/conv_tc_kernel.cuh): `k` is then the program in front of the Convolver; its output rows
  // live in d_cx [V][conv_H + chunk] (history columns in front), d_cxl = their TF32 remainders, d_th / d_tl = Toeplitz(h) hi / lo
  bool conv = false; uint32_t conv_K = 0, conv_H = 0, conv_J = 0, conv_stride = 0, conv_off = 0;
  Array<float> d_cx, d_cxl, d_th, d_tl, d_crows;
  ConvTcMaps conv_maps;
  // two-stage classes are software-pipelined over sub-chunks: dry stage of chunk k+1 (stream) runs beside the FDN of chunk k (stream2)
  Array<float> d_dry2, d_partial2;
  Event e_dry[2], e_fdn[2];
  // banks with several plain classes run the class kernels side by side, each on its own stream (one class alone leaves most
  // warp schedulers with a single warp)
  Stream cstream; Event e_done;
  std::vector<uint32_t> state0;     // initial state, SoA [NS][V]
  // what AudioUnit::reset leaves alone (Lowering::keepS / keepD): state word ranges and delay-line float ranges (per voice), ascending
  std::vector<std::pair<uint64_t, uint64_t>> keep_s, keep_d;
  // Shared readers (Bank::sh_pull): the parameter rows in which some voice reads a Shared, the bank's cell index per voice there (-1: that
  // voice's word there is no reader) and the host image of those rows, [row][V]
  std::vector<uint32_t> sh_rows; std::vector<int32_t> sh_cell; std::vector<uint32_t> sh_img;
  // looping sequencer banks: the reset image also lives on the device (Event<X> resets its unit from it when the event ends, src/sequencer.rs:631-633)
  Array<uint32_t> d_state0; bool state0_stale = true;
  Array<uint32_t> d_params, d_state, d_uniform, d_rowmap;
  Array<float> d_dline, d_partial;
  uint32_t V() const { return (uint32_t)voices.size(); }
};

struct Bank {
  int device = 0; uint32_t out_mode = 0; int nin = 0, nout = 0;
  double sr = DEFAULT_SR; bool dirty = false;
  // voices extracted from a Net: mix in the Net's own association order (0 none, 1 pairwise tree, 2 left fold) and hand the
  // units the Net's f32-rounded sample rate (src/net.rs:132,1323-1328)
  int tree_mix = 0; bool net_rate = false; Array<float> d_rows, d_treepart;
  std::vector<std::unique_ptr<HNode>> nodes;
  std::vector<int> vertex_of_voice;   // banks made from a Net: the Net vertex (NodeId) behind each voice
  std::vector<VoiceClass> classes;
  Stream stream, stream2; Event ev0, ev1, e_begin;
  Array<WaveTableDev> d_wt; Array<float> d_wtdata[6]; WaveTableDev h_wt[6] = {};   // h_wt: host copy of the table directory
  // staging for host-buffer entry points
  Array<float> d_in, d_out, d_mix;
  PinnedArray<float> h_in; MappedArray<float> h_out;   // process() path
  uint64_t launches = 0; float last_ms = 0.0f;
  Array<uint32_t> d_ticket;       // arrival counter of the fused mix-down (short launches)
  bool timing = true;             // record ev0/ev1 around render_device (off on the process() path)
  // event pairs around the DOMINANT kernel of every chunk (the voice program; the FDN kernel of a two-stage class; the tensor-core tiles of
  // a convolver class), on the stream it is launched on: bench.py's roofline divides by this, not by the whole render
  std::vector<Event> dom_ev; size_t dom_n = 0; float last_dom_ms = 0.0f;
  std::string dom_mark(cudaStream_t st);

  // resident process() kernel (dsp/bank_kernel_rt.cuh): a single-class bank that is driven block by block keeps one kernel on the GPU
  // and rings a doorbell per block; every other call on the bank stops it first (state words are saved on the way out)
  MappedArray<RtCtl> rt_ctl; Array<uint32_t> d_rt_relay; Array<float> d_rt_partial;   // (the kernel reads rt_ctl until it exits: ~Bank stops it first)
  bool rt_running = false, in_process = false; uint32_t rt_seq = 1; uint32_t process_streak = 0;
  std::string rt_stop();
  std::string rt_end_streak() { std::string e = rt_stop(); if (e.empty()) process_streak = 0; return e; }   // the next process() calls start a new streak
  std::string rt_process(uint32_t size, const float* in, float* out, bool* served);
  ~Bank();
  uint32_t V() const { return (uint32_t)nodes.size(); }
  double unit_rate() const { return net_rate ? (double)(float)sr : sr; }   // the sample rate the voices' units are given
  std::string init(std::vector<HNode*>& voices, int device, uint32_t out_mode);  // returns "" or error text
  std::string lower_and_upload(bool upload_state);
  std::string set_sample_rate(double sr);
  std::string reset();
  // Sequencer banks (voices made by mk_event): the sequencer clock, replicated on the host with the device's own arithmetic
  // (time += sample_duration * block for every 64-sample block and the tail), live edits and reuse of finished voices
  double seq_time = 0.0;
  double loop_arg = 0.0;              // ReplayMode::Loop(t) of the sequencer the events came from (0: no loop); every event of the bank carries the same t
  double loop_point() const;          // Sequencer::reset :644-650: max(64 samples, t rounded to a sample), +inf without a loop
  void advance_clock(uint64_t n);
  std::string state0_to_device(VoiceClass& c, const uint32_t** out);   // (re)uploads the reset image of an event class of a looping bank
  std::string upload_voice(uint32_t voice, const Lowering& l, bool with_state, const std::vector<uint32_t>* reset_state = nullptr);
  std::string edit_event(uint32_t voice, double end_time, double fade_out);   // Sequencer::edit
  std::string replace_voice(uint32_t voice, HNode* node);                     // a new unit in the slot of a voice of the same class; consumes node
  struct Carry { uint32_t src_s, dst_s, ns; uint64_t src_d, dst_d, nd; };    // state words / delay-line floats of the OLD voice that move into the new one
  std::string regroup(HNode* unit, int at, uint32_t* voice, const Carry* carry = nullptr);   // classes rebuilt around one new / replaced voice, running state of the others kept
  // a unit entering the running bank: `l0` as constructed (what reset() restores), `l` as it runs from now (at the sequencer's clock; `fading`: fading in)
  void lower_entering(HNode* n, Lowering* l0, Lowering* l, bool fading) const;
  std::string crossfade_voice(uint32_t voice, int ease, float fade_time, HNode* unit);   // Net::crossfade: fade the voice to a unit of any class; consumes unit
  std::string remove_voice(uint32_t voice);                                   // Net::remove: the voice carries silence from now on
  std::string add_voice(HNode* unit, uint32_t* voice);                        // grow by one voice, running state of the others preserved; consumes unit
  std::string slot_set(uint32_t voice, int ease, double fade_time, HNode* unit);   // Slot::set: crossfade the voice to a unit of the same class; consumes unit
  // Slot::set while the voice is still fading: the reference parks the update as `latest` (a newer one replaces it) and starts fading to it in the
  // block after the running fade has ended (src/slot.rs:136-161). The bank does the same: the unit waits here, `slot_service` finds the block in
  // which the device's fade ends (the device's own f64 arithmetic, replayed from the voice's fade_phase word), render_device cuts the launch
  // behind that block and arms the waiting unit into the instance that has just gone idle.
  struct SlotLatest { std::unique_ptr<HNode> unit; int ease; double fade_time; };
  std::map<uint32_t, SlotLatest> slot_latest;
  std::map<uint32_t, SlotLatest> xfade_latest;   // the same for Net::crossfade on a vertex that is still fading (`latest` of src/vertex.rs:124-136, :181-245)
  bool has_parked() const { return !slot_latest.empty() || !xfade_latest.empty(); }
  std::string slot_arm_now(uint32_t voice, int ease, double fade_time, HNode* unit, bool force);   // consumes unit; force: also while a fade is running (reset adopts `latest`)
  std::string slot_service(uint64_t n, uint64_t* cut);   // arms parked units whose fade is over; *cut = samples (<= n) after which the first running fade with a parked unit ends
  std::string voice_args(VoiceClass& c, uint32_t len, uint32_t vpc, BankArgs* a);   // class c's part of a launch's arguments; the window starts empty
  std::string render_device_run(uint64_t n, const float* in_dev, uint64_t in_stride, float* out_dev, uint64_t out_stride, float* mix_dev, uint64_t mix_stride);
  std::string push_event(HNode* event, uint32_t* voice);                      // Sequencer::push on a running bank: takes the slot of a finished event of the same class; consumes event
  std::string set(uint32_t voice, const Setting& s);  // AudioUnit::set on one voice of a live bank (parameters only; state continues)
  std::string ensure_staging(uint32_t chunk);
  std::string render_device(uint64_t n, const float* in_dev, uint64_t in_stride, float* out_dev, uint64_t out_stride, float* mix_dev,
                            uint64_t mix_stride);
  std::string render_host(uint64_t n, const float* in, float* out_voices, float* out_mix);
  std::string process(uint32_t size, const float* in, float* out);
  std::string clone_into(Bank& dst) const;
  // Shared controls (graph.h SharedCell). Before a call, sh_pull writes the cells' values into the readers' parameter words; after it,
  // sh_push stores into each written cell the word its last writer in processing order (voice order, then evaluation order) left.
  // A cell is either read or written in one bank: reading what another voice writes would depend on the voice order inside a block.
  std::vector<std::vector<SharedUse>> sh_uses;   // per voice, in evaluation order
  std::vector<SharedRef> sh_cells;               // every cell the voices use (the bank holds a reference)
  std::vector<uint32_t> sh_last;                 // the cells' values at the last sh_pull (empty: compare every reader word)
  struct ShWriter { int cls = -1; uint32_t word = 0, col = 0, voice = 0; };
  std::vector<ShWriter> sh_last_writer;          // per cell: the write-back word stored after a call (cls < 0: the cell is read)
  PinnedArray<uint32_t> sh_stage;   // staging of the reader rows sh_pull copies ([row][V] of every class in turn)
  Event sh_copied; bool sh_pending = false; // recorded behind those copies: the staging is rewritten only after they have landed
  std::string sh_check(uint32_t voice, const std::vector<SharedUse>& uses) const;   // "" or the refusal when `voice` would use `uses`
  std::string sh_rebuild();
  std::string sh_pull();
  std::string sh_push();
  bool sh_writes() const { for (auto& w : sh_last_writer) if (w.cls >= 0) return true; return false; }
};

}  // namespace host
}  // namespace fdsp

/* fundsp_b200 — C ABI of the H100-native voice-bank engine (libfundsp_b200.so).
 *
 * Drop-in boundary for the hot path of SamiPerttu/fundsp v0.23.0: the reference has no FFI; the seam is
 * the Rust trait object `AudioUnit` (src/audiounit.rs:21-95). A Rust host keeps `AudioNode`/`AudioUnit`
 * and the combinator operators (src/combinator.rs:289-488) and binds these entry points (see
 * INTEGRATION.md for the `extern "C"` block and the `trait Lower` walk). Plain pointers and sizes only.
 *
 * Two layers:
 *   1. fdsp_node_*  : construction-time mirror of the reference's graph (one call per primitive node or
 *      combinator; same construction order => same deterministic `ping` hashes, src/audionode.rs:156-161).
 *      Builders CONSUME their child handles (Rust move semantics). NULL is returned on an arity mismatch
 *      (the reference rejects those at compile time) — see fdsp_last_error().
 *   2. fdsp_bank_*  : V voice instances (a Vec of units + mix, SURVEY.md §3.6) evaluated in lockstep on
 *      one GPU; `fdsp_bank_process` == `AudioUnit::process` (src/audiounit.rs:45), `fdsp_bank_render` ==
 *      the `Wave::render` / `Wave::filter` loop (src/wave.rs:441-466, 518-565).
 *
 * Buffers: f32, channel-major. process(): `[channel][64]` like BufferRef/BufferMut (src/buffer.rs:12,156);
 * render(): `[channel][n]`. Voice-major row order for per-voice outputs: row = voice * channels + channel.
 * Errors: every int-returning call returns FDSP_OK or an error code and never throws; the reference's
 * `process` has no error channel, so the Rust shim zero-fills its output on a non-zero status.
 */
#ifndef FUNDSP_B200_H
#define FUNDSP_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct fdsp_node fdsp_node;
typedef struct fdsp_bank fdsp_bank;
typedef struct fdsp_shared fdsp_shared;

enum { FDSP_OK = 0, FDSP_ERR_ARG = 1, FDSP_ERR_CUDA = 2, FDSP_ERR_UNSUPPORTED = 3, FDSP_ERR_ARITY = 4, FDSP_ERR_STATE = 5 };
/* Setting parameter kinds == src/setting.rs:14-31 */
enum { FDSP_P_NULL = 0, FDSP_P_CENTER, FDSP_P_CENTER_Q, FDSP_P_CENTER_Q_GAIN, FDSP_P_VALUE, FDSP_P_COEFFICIENT, FDSP_P_BIQUAD,
       FDSP_P_DELAY, FDSP_P_TIME, FDSP_P_ROUGHNESS, FDSP_P_VARIABILITY, FDSP_P_PAN, FDSP_P_ATTACK_RELEASE, FDSP_P_PHASE,
       FDSP_P_SEED, FDSP_P_INTERVAL };
/* output modes of a bank */
enum { FDSP_OUT_VOICES = 1, FDSP_OUT_MIX = 2 };

const char* fdsp_version(void);
const char* fdsp_last_error(void);          /* thread-local, valid until the next failing call */
int fdsp_device_count(void);                /* number of CUDA devices; 0 when no GPU/driver is usable */

/* ---- graph construction. Leaves: src/prelude.rs constructors; IDs in comments are AudioNode::ID. */
fdsp_node* fdsp_constant(int n, const float* values);          /* Constant<N>   ID 2  (dc / constant) */
fdsp_node* fdsp_pass(void);                                    /* Pass          ID 48 */
fdsp_node* fdsp_multipass(int n);                              /* MultiPass<N>  ID 0  */
fdsp_node* fdsp_sink(int n);                                   /* Sink<N>       ID 1  */
fdsp_node* fdsp_split(int n);                                  /* Split<N>      ID 40 */
fdsp_node* fdsp_multisplit(int m, int n);                      /* MultiSplit    ID 38 */
fdsp_node* fdsp_join(int n);                                   /* Join<N>       ID 41 */
fdsp_node* fdsp_multijoin(int m, int n);                       /* MultiJoin     ID 39 */
fdsp_node* fdsp_reverse(int n);                                /* Reverse<N>    ID 45 */
fdsp_node* fdsp_sine(void);                                    /* Sine<f32>     ID 21 src/oscillator.rs:18 */
fdsp_node* fdsp_wavesynth(int table, int outputs);             /* WaveSynth<N>  ID 34; table 0 saw 1 square 2 triangle 3 organ 4 soft_saw 5 hammond */
fdsp_node* fdsp_noise(void);                                   /* Noise         ID 20 src/noise.rs:170 */
fdsp_node* fdsp_fixed_svf(int mode, float cutoff, float q, float gain); /* FixedSvf ID 43; mode 0 lowpass 1 highpass 2 bandpass 3 notch 4 peak 5 allpass 6 bell 7 lowshelf 8 highshelf */
fdsp_node* fdsp_svf(int mode, float cutoff, float q, float gain);       /* Svf ID 36 (audio, cutoff, q[, gain] inputs) */
/* prelude64 (F = f64): the same nodes with f64 internal state, as `fundsp::prelude64` builds them. Arguments and node inputs/outputs stay
   f32 and are widened to f64; coefficients are computed in f64 (libm tan), the sample rate is the f64 one the node receives. */
fdsp_node* fdsp_sine_f64(void);                                /* Sine<f64>     ID 21: f64 phase; output sin(phase as f32 * TAU) */
fdsp_node* fdsp_fixed_svf_f64(int mode, float cutoff, float q, float gain); /* FixedSvf<f64, M> ID 43; modes as fdsp_fixed_svf */
fdsp_node* fdsp_svf_f64(int mode, float cutoff, float q, float gain);       /* Svf<f64, M> ID 36 (audio, cutoff, q[, gain] inputs) */
fdsp_node* fdsp_biquad_f64(float a1, float a2, float b0, float b1, float b2); /* Biquad<f64> ID 15 */
fdsp_node* fdsp_butterpass_f64(float cutoff, int inputs);      /* ButterLowpass<f64, U1|U2> ID 16 (inputs 1 = butterpass_hz) */
fdsp_node* fdsp_resonator_f64(float center, float q, int inputs); /* Resonator<f64, U1|U3> ID 17 (inputs 1 = resonator_hz) */
fdsp_node* fdsp_onepole_f64(int kind, float param, int inputs); /* the fdsp_onepole kinds 0..4 with F = f64 (Lowpole, Highpole, Allpole, DCBlock, Pinkpass) */
fdsp_node* fdsp_biquad(float a1, float a2, float b0, float b1, float b2); /* Biquad<f32> ID 15 */
fdsp_node* fdsp_biquad_bank(void);                             /* BiquadBank<f32x8> ID 98 */
fdsp_node* fdsp_butterpass(float cutoff, int inputs);          /* ButterLowpass ID 16 (inputs 1 = butterpass_hz) */
fdsp_node* fdsp_resonator(float center, float q, int inputs);  /* Resonator     ID 17 (inputs 1 = resonator_hz) */
fdsp_node* fdsp_moog(float cutoff, float q, int inputs);       /* Moog<f32,U1|U3> ID 60 */
fdsp_node* fdsp_fir(int n, const float* weights);              /* Fir<N>        ID 52 */
fdsp_node* fdsp_tick(int n);                                   /* Tick<N>       ID 9  */
fdsp_node* fdsp_delay(double seconds);                         /* Delay         ID 13 */
fdsp_node* fdsp_allnest(float coefficient, fdsp_node* x, int inputs); /* AllNest ID 83 */
fdsp_node* fdsp_phase_osc(int kind);                           /* kind 0 Ramp ID 94, 1 PolySaw 95, 2 PolySquare 96, 3 PolyPulse 97 (src/oscillator.rs:440-760) */
fdsp_node* fdsp_reverb3(double time, double diffusion, fdsp_node* filter); /* Reverb<F> ID 85 src/reverb.rs:156 (reverb3_stereo); consumes the 1->1 loop filter */
fdsp_node* fdsp_feedback_unit(double delay, fdsp_node* x);   /* FeedbackUnit ID 79 src/feedback.rs:347: feedback with integrated delay (>= 1 sample) */
fdsp_node* fdsp_convolve(const float* response, int n);       /* Convolver ID 100 src/convolve.rs:14: linear convolution with `response` (shared by all voices that pass the same one) */
fdsp_node* fdsp_onepole(int kind, float param, int inputs);   /* src/filter.rs: kind 0 Lowpole ID 18 (cutoff), 1 Highpole 47 (cutoff), 2 Allpole 46 (delay), 3 DCBlock 22 (cutoff), 4 Pinkpass 26; inputs 2 = audio-rate parameter */
fdsp_node* fdsp_shaper(int kind, float p0, float p1);         /* Shaper<S> ID 42 src/shape.rs: kind 0 Clip(h) 1 ClipTo(lo,hi) 2 Tanh(h) 3 Softsign(h) 4 Crush(levels) 5 SoftCrush(levels) 6 Atan(h) */
fdsp_node* fdsp_follow(int asymmetric, float attack, float release); /* Follow ID 24 (asymmetric 0: response time = attack) / AFollow ID 29, src/follow.rs */
fdsp_node* fdsp_morph(float cutoff, float q);                  /* Morph ID 62 src/svf.rs:1040: inputs (audio, cutoff, q, morph -1..1) */
fdsp_node* fdsp_rez(float bandpass, float cutoff, float q, int inputs); /* Rez ID 75 src/rez.rs: bandpass 0 = lowrez, 1 = bandrez; inputs 1 or 3 (audio, cutoff, q) */
fdsp_node* fdsp_chaos(int kind);                               /* kind 0 Rossler ID 73, 1 Lorenz ID 74 (src/oscillator.rs:318-438); input = frequency */
fdsp_node* fdsp_declick(float duration);                       /* Declick ID 23 src/dynamics.rs:245: smooth fade-in over `duration` seconds */
fdsp_node* fdsp_oversample(fdsp_node* x);                      /* Oversampler<X> ID 51 src/oversample.rs (`oversample`): x at 2x the sample rate between 43-tap minimum-phase halfbands; consumes x (inputs <= outputs) */
fdsp_node* fdsp_monitor(void);                                 /* Monitor ID 56 src/dynamics.rs:441 (`monitor(&shared, meter)`): the audio passes through; the Shared it feeds stays host-side (read the level with a `meter` voice output instead) */
/* Envelope<F, E, R> ID 14 src/envelope.rs:14 (`envelope`, `lfo`; interval 0.002): the closure E crosses the ABI as a HOST callback. It is
   called when the graph is lowered (bank creation, sample-rate change, settings) — never while rendering — at exactly the jittered sample
   points the reference would evaluate it at (they depend only on the node's hash and the interval), for points up to `horizon` seconds;
   later the last value holds. time_f64: F = f64, else f32 (t is then an f32 value). f and user must outlive the node and its bank. */
typedef void (*fdsp_envelope_fn)(double t, double* out /* [outputs] */, void* user);
fdsp_node* fdsp_envelope(double interval, int outputs, int time_f64, fdsp_envelope_fn f, void* user, double horizon);
/* One event of a Sequencer (src/sequencer.rs:319-345 `push`) as a voice: the generator x sounds from start to end seconds (sample
   accurate, the reference's rounding), with fade-in / fade-out of the given lengths; fade_ease 0 Fade::Power, 1 Fade::Smooth. A bank
   of events IS the sequencer: its mix output is Sequencer::process. Consumes x. */
fdsp_node* fdsp_event(fdsp_node* x, double start, double end, int fade_ease, double fade_in, double fade_out);
/* The same for a sequencer made with ReplayMode::Loop(loop_seconds) (src/sequencer.rs:219-229; loop_seconds == 0: fdsp_event): the event
   keeps the sequencer's loop point (>= 64 samples, rounded to a sample, :644-650) and replays every period — an event that straddles the
   loop point continues into the next period shifted by it, a finished one is reset (its unit back to its construction state, :622-639)
   and starts again. All voices of a looping bank are events with the same loop_seconds, pushed before the first render; the block path
   is the reference's AS WRITTEN: the samples of a 64-block behind the wrap are rendered but not delivered (:845-872). */
fdsp_node* fdsp_event_loop(fdsp_node* x, double start, double end, int fade_ease, double fade_in, double fade_out, double loop_seconds);
fdsp_node* fdsp_limiter(int channels, float attack, float release); /* Limiter<N> ID 25 src/dynamics.rs:128 (`limiter`, `limiter_stereo`): look-ahead = attack seconds */
fdsp_node* fdsp_meter(int kind, double timescale);             /* MeterNode ID 61 src/dynamics.rs:316: kind 0 Meter::Sample, 1 Peak(timescale), 2 Rms(timescale) */
/* WavePlayer ID 65 src/wave.rs:739 (`playwave`, `playwave_at`): `samples` = wave.channel(ch) (copied); plays [start, end), then jumps to
   loop_point (-1 = none, silence after the end). Voices playing the same samples share one device copy. */
fdsp_node* fdsp_playwave(const float* samples, uint64_t length, uint64_t start, uint64_t end, int64_t loop_point);
fdsp_node* fdsp_resample(fdsp_node* x);                        /* Resample<X> ID 69 src/resample.rs:210 (`resample`): input = speed; consumes the generator x */
fdsp_node* fdsp_phase_synth(int kind);                         /* PhaseSynth ID 35 src/wavetable.rs:361: input = phase, table kind as fdsp_wavesynth */
fdsp_node* fdsp_pulse(void);                                   /* PulseWave ID 44 src/wavetable.rs:439 (`pulse()`): inputs (frequency, width 0..1) */
fdsp_node* fdsp_mixer(int inputs, int outputs, const float* matrix); /* Mixer<M,N> ID 84 src/pan.rs:95: matrix[output * inputs + input] */
fdsp_node* fdsp_rotate(float angle, float gain);               /* `rotate(angle, gain)` src/prelude.rs:2876: the 2x2 Mixer of a stereo rotation */
/* nonlinear biquads src/biquad.rs:494-920: fb 1 = FbBiquad 88 / FixedFbBiquad 90, 0 = DirtyBiquad 89 / FixedDirtyBiquad 91; mode 0 resonator,
   1 lowpass, 2 highpass, 3 bell; shape kind + (p0, p1) as in fdsp_shaper; inputs 1 = fixed (center, q, gain given), 3 (4 for bell) = audio rate */
fdsp_node* fdsp_nl_biquad(int fb, int mode, int shape, float p0, float p1, int inputs, float center, float q, float gain);
/* Adaptive<S> src/shape.rs:156-200 (`Adaptive::new(timescale, inner)`): the input is divided by its running RMS estimate (halfway to a new
   level in `timescale` seconds, taken as f32) before the inner shape, one of the fdsp_shaper kinds 0..6 with its (p0, p1). The estimate
   starts at 0 in a new unit and at 1e-3 after a reset. In Shaper<Adaptive> the smoothing follows the sample rate; the nonlinear biquads
   keep the one computed at 44.1 kHz (their set_sample_rate does not reach the shape). NULL with the reason for an inner kind outside
   0..6 (an Adaptive or a shape_fn cannot be nested) or a timescale that is not positive. */
fdsp_node* fdsp_shaper_adaptive(double timescale, int inner_kind, float p0, float p1);
fdsp_node* fdsp_nl_biquad_adaptive(int fb, int mode, double timescale, int inner_kind, float p0, float p1, int inputs, float center, float q, float gain);
fdsp_node* fdsp_var(float value);                              /* Var ID 68 src/shared.rs:84: control value, changed with Setting::value (fdsp_node_set / fdsp_bank_set) */
/* Shared src/shared.rs:47-81: a 32-bit cell set and read from any thread with relaxed atomics (an f32 bit pattern). Reference counted:
   fdsp_shared_free drops the caller's reference; every node built on the cell, and every bank holding such a node, keeps one of its own
   (clones share the cell, as an Arc clone does). fdsp_shared_wrap uses memory the caller owns — the AtomicU32 behind a Rust Shared,
   `Shared::get_shared().as_ptr()`; `release(user)` (may be NULL) is called once when the last reference is dropped, which is when the
   memory may go (the Rust binding passes `Arc::into_raw` of a clone and drops it there).
   Banks read readers' cells once before each process / render call: a set between two calls holds for the whole next call. After a
   call the bank stores into each written cell what its last writer in processing order stores (the last voice in bank order, within it
   the last writer in evaluation order). A bank in which one cell is both read and written is refused with FDSP_ERR_UNSUPPORTED. */
fdsp_shared* fdsp_shared_new(float value);
fdsp_shared* fdsp_shared_wrap(uint32_t* cell, void (*release)(void* user), void* user);
void fdsp_shared_free(fdsp_shared* s);
void fdsp_shared_set(fdsp_shared* s, float value);
float fdsp_shared_get(const fdsp_shared* s);
fdsp_node* fdsp_var_shared(fdsp_shared* s);                                     /* Var ID 68: var(&shared) */
fdsp_node* fdsp_monitor_shared(fdsp_shared* s, int kind, double timescale);     /* Monitor ID 56: monitor(&shared, meter), kind as fdsp_meter */
/* VarFn ID 70 (`var_fn(&shared, f)`): the closure, as text in the language of fdsp_map with one parameter |x| (the cell's value), returning
   `outputs` values; evaluated once per call with the value the call reads. NULL with the reason as for fdsp_map. */
fdsp_node* fdsp_var_fn(fdsp_shared* s, int outputs, const char* closure, int ncaptures, const char* const* names, const float* values);
fdsp_node* fdsp_timer(fdsp_shared* s);                                          /* Timer ID 57: timer(&shared); sets the cell to 0 now, and on reset */
fdsp_node* fdsp_dsf(int inputs, float harmonic_spacing, float roughness); /* Dsf<N> ID 55 src/oscillator.rs:114 (dsf_saw / dsf_square) */
fdsp_node* fdsp_mls(int bits);                                 /* Mls           ID 19 src/noise.rs:100 */
fdsp_node* fdsp_impulse(int n);                                /* Impulse<N>    ID 81 */
fdsp_node* fdsp_tap(int taps, int linear, float min_delay, float max_delay); /* Tap<N> ID 50 / TapLinear<N> ID 54 */
fdsp_node* fdsp_feedback2(fdsp_node* x, fdsp_node* y, int hadamard);         /* Feedback2 ID 66 (feedback2 / fdn2) */
fdsp_node* fdsp_pan(float value);                              /* Panner<U1>    ID 49 */
fdsp_node* fdsp_panner(void);                                  /* Panner<U2>    ID 49 */
fdsp_node* fdsp_adsr_live(float attack, float decay, float sustain, float release); /* EnvelopeIn ID 53 + src/adsr.rs closure */
/* Closures of the signal, run per sample on the device. The closure is TEXT in a subset of Rust closure syntax (DESIGN.md §2), e.g.
   "|x| tanh(x[0] * drive)"; any other free identifier is a captured value, passed as (names[k], values[k]) pairs. The parsed closure
   becomes part of the voice's class (literals included); captured values are per-voice, so voices that differ only in them share a
   class. Map has 0-8 inputs and 1-8 outputs; a tuple value is a multi-output closure. On failure these return NULL with the reason and
   its column in fdsp_last_error(): reasons that begin "<node>: arity mismatch" are arity errors (the reference rejects them at compile
   time); every other refusal (syntax, an unsupported function, a capture that does not occur in the text, an identifier without a
   value) is an argument error. Only the envelopes have a settable parameter: fdsp_envelope_in and fdsp_envelope_text take Setting::interval. */
fdsp_node* fdsp_map(int inputs, int outputs, const char* closure, int ncaptures, const char* const* names, const float* values);        /* Map ID 5 src/audionode.rs:1328 (`map`): |x| with x[0..inputs) */
fdsp_node* fdsp_shape_fn(const char* closure, int ncaptures, const char* const* names, const float* values);                          /* Shaper<ShapeFn> ID 42 src/shape.rs:33 (`shape_fn`): |x| with a scalar x */
fdsp_node* fdsp_envelope_in(double interval, int inputs, int outputs, const char* closure, int ncaptures, const char* const* names, const float* values); /* EnvelopeIn<f32> ID 53 src/envelope.rs:185 (`envelope_in`, `envelope2`, `envelope3`, `lfo_*`; interval 0.002): |t, i| with a frame i[0..inputs), or |t, x1, .., xN| with one scalar per input */
/* Envelope<f32, E, R> ID 14 src/envelope.rs:14 (`envelope`, `lfo`; interval 0.002) with the closure E as TEXT |t| of time alone, 1-8
   outputs: the device evaluates it at the reference's jittered sample points (the same points as fdsp_envelope's callback), so it has no
   horizon and stores no table of values. The closure computes in f32; for F = f64 time use fdsp_envelope's callback. */
fdsp_node* fdsp_envelope_text(double interval, int outputs, const char* closure, int ncaptures, const char* const* names, const float* values);
/* System ID 67 src/system.rs (`update(x, dt, f)`): f is `|t, dt, x| ..` whose body is `let`s and unconditional statements
   `x.set(Setting::KIND(args)[.left() | .right() | .index(N)]*);` with KIND center, center_q, center_q_gain, value, pan or biquad; run at the
   start of a block every ~dt seconds (and at time 0). Consumes x. NULL with the reason as for fdsp_map. A `set` that reaches a node other
   than FixedSvf, the fixed ButterLowpass / Biquad, the fixed one-poles, Constant or Panner<U1> and that the node does not ignore (a Resonator
   ignores every setting) makes the bank FDSP_ERR_UNSUPPORTED. */
fdsp_node* fdsp_update(fdsp_node* x, float dt, const char* closure, int ncaptures, const char* const* names, const float* values);
/* combinators (src/combinator.rs:289-488; src/audionode.rs) */
fdsp_node* fdsp_pipe(fdsp_node* x, fdsp_node* y);              /* x >> y  Pipe   ID 6  */
fdsp_node* fdsp_stack(fdsp_node* x, fdsp_node* y);             /* x | y   Stack  ID 7  */
fdsp_node* fdsp_branch(fdsp_node* x, fdsp_node* y);            /* x ^ y   Branch ID 8  */
fdsp_node* fdsp_bus(fdsp_node* x, fdsp_node* y);               /* x & y   Bus    ID 10 */
fdsp_node* fdsp_thru(fdsp_node* x);                            /* !x      Thru   ID 12 */
fdsp_node* fdsp_binop(int op, fdsp_node* x, fdsp_node* y);     /* op 0 x+y, 1 x-y, 2 x*y   Binop ID 3 */
fdsp_node* fdsp_unop(int kind, float scalar, fdsp_node* x);    /* kind 0 -x, 1 x+s, 2 s-x, 3 x*s   Unop ID 4 */
fdsp_node* fdsp_multi(int kind, int op, int n, fdsp_node* const* nodes); /* kind 28 MultiBus, 30 MultiStack, 31 Reduce(op), 33 MultiBranch, 32 Chain */
fdsp_node* fdsp_feedback(fdsp_node* x, int hadamard);          /* Feedback<N,X,FrameId|FrameHadamard> ID 11 */
/* Net (src/net.rs:118-146, 204-213, 472-640): dynamic DAG of units; vertex ids are indices in push order */
fdsp_node* fdsp_net_new(int inputs, int outputs);                 /* Net::new           ID 63 */
int fdsp_net_push(fdsp_node* net, fdsp_node* unit);               /* Net::push -> vertex index (consumes unit), < 0 on error */
int fdsp_net_connect(fdsp_node* net, int source, int source_port, int target, int target_port);   /* Net::connect */
int fdsp_net_connect_input(fdsp_node* net, int global_input, int target, int target_port);        /* Net::connect_input */
int fdsp_net_connect_output(fdsp_node* net, int source, int source_port, int global_output);      /* Net::connect_output */
int fdsp_net_pass_through(fdsp_node* net, int global_input, int global_output);                   /* Net::pass_through */
int fdsp_net_size(const fdsp_node* net);
/* An<X> builder methods (src/combinator.rs:263-276) and generic Setting (src/setting.rs:52-211) */
int fdsp_node_phase(fdsp_node* n, float phase);
int fdsp_node_seed(fdsp_node* n, uint64_t seed);
int fdsp_node_set(fdsp_node* n, int kind, const float* values, int nvalues, uint64_t seed, const int64_t* address_pairs, int naddress);
int fdsp_node_inputs(const fdsp_node* n);
int fdsp_node_outputs(const fdsp_node* n);
uint64_t fdsp_node_id(const fdsp_node* n);
uint64_t fdsp_node_ping(fdsp_node* n, int probe, uint64_t hash);            /* AudioNode::ping */
int fdsp_node_leaf_hashes(fdsp_node* n, uint64_t* out, int max);            /* hashes handed to leaves by the constructor ping, in order */
int fdsp_node_set_sample_rate(fdsp_node* n, double sample_rate);             /* AudioNode::set_sample_rate on a graph that is not in a bank yet */
int fdsp_node_signature(const fdsp_node* n, char* out, int max);            /* device program type expression */
/* the words the device program of this node consumes, in load order: per-voice parameters P, initial state S, class-uniform U
   (host-only introspection; counts are returned even when the buffers are too small or NULL) */
int fdsp_node_lowering(const fdsp_node* n, uint32_t* P, int maxp, uint32_t* S, int maxs, uint32_t* U, int maxu, int* np, int* ns, int* nu);
int64_t fdsp_node_delay_floats(const fdsp_node* n);                           /* per-voice delay-line storage (floats) of the device program; -1 on error */
fdsp_node* fdsp_node_clone(const fdsp_node* n);
void fdsp_node_free(fdsp_node* n);
/* wavetable introspection (host builder, src/wavetable.rs:82-123) */
int fdsp_wavetable_count(int table);
int fdsp_wavetable_info(int table, int index, float* pitch, int* length);
const float* fdsp_wavetable_data(int table, int index);

/* ---- voice banks */
/* Takes ownership of `voices`. Voices may belong to several structural classes (dynamic Net of mixed
 * graphs): each class becomes one fused kernel. All voices must agree on inputs() and outputs(). */
int fdsp_bank_create(fdsp_node* const* voices, uint32_t nvoices, int device, uint32_t out_mode, fdsp_bank** out);
/* A voice-separable Net (voice vertices + the adder trees Net::bus builds) becomes a bank whose mix-down follows the
 * Net's own association order bit for bit; voices get the hashes of Net::ping (src/net.rs:1383-1389). Consumes `net`. */
int fdsp_bank_create_from_net(fdsp_node* net, int device, uint32_t out_mode, fdsp_bank** out);
/* banks made from a Net: voice index of Net vertex `vertex` (the NodeId of Net::push), -1 if it is not a voice. With it
   `net.set(setting.node(id))` (src/net.rs:1159-1169) becomes fdsp_bank_set(bank, fdsp_bank_voice_of_vertex(bank, id), ...) */
int fdsp_bank_voice_of_vertex(const fdsp_bank* b, int vertex);
void fdsp_bank_destroy(fdsp_bank* b);
int fdsp_bank_clone(const fdsp_bank* b, fdsp_bank** out);                   /* deep copy incl. device state (dyn_clone) */
uint32_t fdsp_bank_voices(const fdsp_bank* b);
int fdsp_bank_inputs(const fdsp_bank* b);                                   /* shared (bus) input channels */
int fdsp_bank_voice_outputs(const fdsp_bank* b);                            /* channels per voice */
int fdsp_bank_outputs(const fdsp_bank* b);                                  /* AudioUnit::outputs(): mix: channels; voices: V*channels */
int fdsp_bank_set_sample_rate(fdsp_bank* b, double sample_rate);            /* AudioUnit::set_sample_rate */
/* Programs of graph classes outside the ahead-of-time table are compiled with NVRTC on first use and kept in an on-disk cache
   ($FDSP_JIT_CACHE, default jit_cache/ next to the library; "off" disables it). fdsp_jit_precompile fills the cache WITHOUT a GPU:
   `signature` is fdsp_node_signature's text, mode 0 the layout unit every class needs, 1..3 the kernel variant of FDSP_OUT_* with
   (table_variant 1) or without the shared-memory wavetable stage. fdsp_jit_cache_stats: units served from disk / compiled in this process. */
int fdsp_jit_precompile(const char* signature, int mode, int table_variant);
void fdsp_jit_cache_stats(int* hits, int* nvrtc_runs);
/* WAV edge (reference src/write.rs:24-116): `planar[c * stride + i]` -> Wave::write_wav16 (bits 16: round(clamp11(x) * 32767.49)) or
   Wave::write_wav32 (bits 32: IEEE float) byte for byte — to a file, or into `out` (returns the byte count, also when out is NULL or
   too small; -1 on error). fdsp_wave_load reads the two layouts back (16-bit samples / 32768); call it with planar = NULL to get the
   sizes first. */
int fdsp_wave_save(const char* path, const float* planar, uint32_t channels, uint64_t length, uint64_t stride, double sample_rate, int bits);
int64_t fdsp_wave_encode(uint8_t* out, uint64_t max, const float* planar, uint32_t channels, uint64_t length, uint64_t stride, double sample_rate, int bits);
int fdsp_wave_load(const char* path, float* planar, uint64_t max_floats, uint32_t* channels, uint64_t* length, double* sample_rate);
/* Sequencer banks (voices made by fdsp_event; the bank's mix output is Sequencer::process, src/sequencer.rs:768-843).
   fdsp_bank_edit_event = Sequencer::edit (:441-483): new end time and fade-out of one event, effective from the next block.
   fdsp_bank_push_event = Sequencer::push on a running sequencer (:319-360): the event takes over the slot of a FINISHED event of the
   same graph class (same type expression and class-uniform words) and starts its clock at the bank's current time; `*voice` receives
   the slot. When no such slot is free the bank GROWS by one voice (fdsp_bank_add_voice: the running state and delay lines of all
   voices are read back, the classes rebuilt — the newcomer may found a new class, compiled first — and the state written into the
   new layout; O(bank state), not for the audio thread; banks with an FDN-reverb class or made from a Net cannot grow in place).
   fdsp_bank_replace_voice = Net::replace (src/net.rs:460-470) / a new unit in a voice's place, fresh state: any unit of the bank's arity. A unit
   of the voice's own graph class is written into its slot; a unit of another class moves the voice to that class (compiled first if new) —
   the classes are regrouped around it, every other voice keeps its running state and, in a bank made from a Net, the voice keeps its
   place in the Net's mix order. fdsp_bank_remove_voice = Net::remove (:351-404, connections replaced with zeros): the voice carries
   silence from now on. Both are the slow path (O(bank state)), like add_voice. All consume their node argument.
   fdsp_bank_time = Sequencer::time (seconds rendered since reset). */
int fdsp_bank_edit_event(fdsp_bank* b, uint32_t voice, double end_time, double fade_out);
int fdsp_bank_push_event(fdsp_bank* b, fdsp_node* event, uint32_t* voice);
int fdsp_bank_replace_voice(fdsp_bank* b, uint32_t voice, fdsp_node* unit);
/* Net::crossfade (src/net.rs:480-504): the voice fades from its unit to `unit` — any graph class of the bank's arity — over fade_time seconds
   with the curve fade_ease (0 Fade::Power, 1 Fade::Smooth), the reference's f32 vertex arithmetic (src/vertex.rs:138-229), and is `unit` alone
   afterwards. Both programs run in the voice while the fade lasts (class Xfade<old, new>, compiled first if new; the old unit's running state
   and delay lines are carried into it; slow path like replace_voice). A further crossfade of a voice that is still fading waits as the vertex's
   `latest` edit (a newer one replaces it) and starts in the block after the running fade has ended, like src/vertex.rs:124-136,203-218: the bank
   finds that block and cuts its launch there. A bank reset leaves the voice at `unit`. Consumes unit. */
int fdsp_bank_crossfade_voice(fdsp_bank* b, uint32_t voice, int fade_ease, float fade_time, fdsp_node* unit);
int fdsp_bank_add_voice(fdsp_bank* b, fdsp_node* unit, uint32_t* voice);
int fdsp_bank_remove_voice(fdsp_bank* b, uint32_t voice);
double fdsp_bank_time(const fdsp_bank* b);
/* Slot / SlotBackend (src/slot.rs): fdsp_slot(unit) is a voice whose unit can be replaced while the bank runs; fdsp_bank_slot_set is
   Slot::set(fade, fade_time, unit): the voice crossfades to `unit` over fade_time seconds (fade 0 Power, 1 Smooth) with the reference's
   block arithmetic. No new program is built: `unit` must be of the voice's graph class (same type expression and class-uniform words,
   e.g. the same instrument with other parameters), else FDSP_ERR_UNSUPPORTED. A set while a previous crossfade of that voice is still
   running waits as `latest` (a newer one replaces it) and starts in the block after the running fade has ended; a reset adopts it
   (src/slot.rs:136-172). Both consume their node argument. */
fdsp_node* fdsp_slot(fdsp_node* unit);
int fdsp_bank_slot_set(fdsp_bank* b, uint32_t voice, int fade_ease, double fade_time, fdsp_node* unit);
int fdsp_bank_reset(fdsp_bank* b);                                          /* AudioUnit::reset */
/* AudioUnit::set (src/audiounit.rs:62) on voice `voice` of a live bank: same encoding as fdsp_node_set. Parameters change at
   once, running state continues; FDSP_ERR_UNSUPPORTED when the setting would change a delay length (rebuild the bank). */
int fdsp_bank_set(fdsp_bank* b, uint32_t voice, int kind, const float* values, int nvalues, uint64_t seed, const int64_t* address_pairs, int naddress);
/* fdsp_bank_set on n entries in one call: entry j sets voice voices[j] (j when voices is NULL) to values[j*nvalues .. +nvalues) with seed
   seeds[j] (0 when seeds is NULL); one setting kind and one address for all. The same as calling fdsp_bank_set for j = 0, 1, .. n-1:
   entries of one voice apply in order, and on the first entry that call would refuse, this one returns its error with *failed_entry = j
   (the entries before j applied, the rest not; n on success). Values are host memory. The parameter words reach the device in one copy
   and one launch per class the entries touch. */
int fdsp_bank_set_voices(fdsp_bank* b, int kind, const uint32_t* voices, uint32_t n, const float* values, int nvalues, const uint64_t* seeds,
                         const int64_t* address_pairs, int naddress, uint32_t* failed_entry);
/* fdsp_bank_set_voices with the values in device memory: values_dev is [n][nvalues] f32 on the bank's device, and the coefficients are
   computed there, one kernel per class the entries touch. voices (NULL: entry j is voice j) is host memory. `stream` is the cudaStream_t
   that writes the values (NULL: the legacy default stream): the bank waits for the work queued on it, and it waits for the bank's kernels,
   so the caller may overwrite the values in stream order once this returns. Asynchronous: the sets take effect from the next process or
   render call, and leave the bank exactly as fdsp_bank_set_voices with the same values would (entries of one voice: the last one wins).
   The node an address reaches must be a FixedSvf (center, center_q, center_q_gain), the fixed ButterLowpass (center), the fixed Biquad
   (biquad), a fixed Lowpole / Highpole / DCBlock (center), a Constant (value) or a Panner<U1> (pan); an address that leads nowhere, or a
   setting the node ignores, changes nothing. Values are not checked.
   Unlike fdsp_bank_set_voices, a refusal applies NO entry (the host never sees the values, so every entry is checked first):
   *failed_entry = the first refused entry (n on success), FDSP_ERR_ARG for a voice out of range, FDSP_ERR_UNSUPPORTED for a voice whose
   address reaches any other node that does not ignore the setting (checked voice by voice: voices of one class can hold different nodes,
   e.g. dc and var), a Slot, a crossfading vertex, a System or a Net, or uses .node(id), or whose node's parameter words share a row with
   other voices' Shared readers (var(&shared) in the same class). The host graphs take the device's sets before any call that reads
   them; process and the renders never wait for that, except when a parked Slot / crossfade update falls due in them. */
int fdsp_bank_set_voices_device(fdsp_bank* b, int kind, const uint32_t* voices, uint32_t n, const float* values_dev, int nvalues,
                                const int64_t* address_pairs, int naddress, void* stream, uint32_t* failed_entry);
int fdsp_bank_allocate(fdsp_bank* b, uint64_t max_render_samples);          /* AudioUnit::allocate: later calls do not allocate */
/* AudioUnit::process: size <= 64; host buffers in [inputs][64], out [outputs][64]; size 0 is a no-op */
int fdsp_bank_process(fdsp_bank* b, uint32_t size, const float* in, float* out);
/* Wave::render / Wave::filter: host buffers; in [inputs][n] or NULL; out_voices [V*channels][n] or NULL; out_mix [channels][n] or NULL */
int fdsp_bank_render(fdsp_bank* b, uint64_t n, const float* in, float* out_voices, float* out_mix);
/* same with device-resident buffers (strides in floats), asynchronous on the bank's stream */
int fdsp_bank_render_device(fdsp_bank* b, uint64_t n, const float* in_dev, uint64_t in_stride, float* out_voices_dev, uint64_t voices_stride,
                            float* out_mix_dev, uint64_t mix_stride);
int fdsp_bank_sync(fdsp_bank* b);
/* ---- multi-GPU mix-down (SURVEY.md §8e; csrc/host/group.h). Voices shard across ranks: one bank per GPU (one process per GPU, or
   several banks in one process), no data-path collective — the ONE exchange step is the sum of the per-GPU partial mixes. It runs
   below this ABI over NCCL / NVLink on the bank's own stream, so `render_reduced` is to a sharded bank what `Wave::render` of
   "a Vec of units + a sum" (reference src/wave.rs:441-466) is to one: the root rank receives the finished mix.
   Default association: the partials are gathered on the root and added in RANK ORDER ((p0 + p1) + p2) + ..., independent of NCCL's
   algorithm choice (FDSP_GROUP_REDUCE=nccl: plain ncclReduce). The 128-byte unique id comes from rank 0 and is handed to the other
   ranks by the host (a file, a socket, MPI, torch.distributed ...), like ncclGetUniqueId / ncclCommInitRank. */
typedef struct fdsp_group fdsp_group;
int fdsp_group_unique_id(void* id, uint64_t bytes);                          /* bytes >= 128 */
int fdsp_group_create(int nranks, int rank, const void* id, int device, fdsp_group** out);   /* collective: every rank calls it */
void fdsp_group_destroy(fdsp_group* g);
int fdsp_group_rank(const fdsp_group* g);
int fdsp_group_size(const fdsp_group* g);
/* renders `samples` of this rank's bank (FDSP_OUT_MIX) and reduces; out_mix [channels][samples] (host) is written on `root` only */
int fdsp_bank_render_reduced(fdsp_bank* b, fdsp_group* g, uint64_t samples, const float* in, float* out_mix, int root);
/* device form: mix_dev [channels][mix_stride] holds this rank's partial (e.g. from fdsp_bank_render_device) and, on the root, the sum
   afterwards; enqueued on the bank's stream */
int fdsp_bank_reduce_device(fdsp_bank* b, fdsp_group* g, uint64_t samples, float* mix_dev, uint64_t mix_stride, int root);
void* fdsp_bank_stream(fdsp_bank* b);                                       /* cudaStream_t the bank launches on */
/* introspection */
int fdsp_bank_num_classes(const fdsp_bank* b);
int fdsp_bank_class_info(const fdsp_bank* b, int cls, char* signature, int max, uint32_t* voices, uint32_t* state_words, uint32_t* param_words, uint64_t* delay_floats);
int fdsp_bank_class_stages(const fdsp_bank* b, int cls);                    /* warp stages of the class's stage-pipelined kernel (csrc/dsp/bank_kernel_st.cuh); 1 = it has none */
uint64_t fdsp_bank_launch_count(const fdsp_bank* b);                        /* kernels launched so far */
float fdsp_bank_last_kernel_ms(const fdsp_bank* b);                         /* CUDA-event time of the voice kernels of the last render_device call */
float fdsp_bank_last_dominant_ms(const fdsp_bank* b);                       /* of that, the dominant kernel alone (voice program | FDN kernel | tensor-core tiles), summed over chunks and classes */

#ifdef __cplusplus
}
#endif
#endif

//! GPU voice banks for FunDSP graphs: binding of `libfundsp_b200.so` (C ABI: include/fundsp_b200.h).
//!
//! Written against fundsp v0.23.0. NOT compiled in the fundsp_b200 repository (no Rust toolchain in its build image); the C++ and
//! Python mirrors of this file are what its tests run. Lives in the crate (`src/gpu.rs`, feature `gpu`) because lowering reads
//! construction-time parameters that are private fields; it needs these `pub(crate)` accessors added next to the fields:
//!   Sine::<F>::initial_phase() -> Option<F>         (oscillator.rs:25)     WaveSynth::initial_phase() / table_kind() (wavetable.rs:258)
//!   Noise::seed() -> Option<u64>                    (noise.rs:175)         FixedSvf::<F, M>::params() -> &SvfParams<F> (svf.rs:867)
//!   Moog::cutoff_q() -> (f32, f32)                  (moog.rs:20-34)        Fir::weights() -> &[f32]                  (fir.rs:15)
//!   Delay::length_seconds() -> f64                  (delay.rs:69)          Panner::<U1>::pan_value() -> f32          (pan.rs:19)
//!   Unop scalar: FrameAddScalar / FrameMulScalar / FrameNegAddScalar ::scalar() (audionode.rs:1114,1155,1197)
//!   Resonator::<F, N>::center_q() -> (F, F)         (biquad.rs:310-318)    ButterLowpass::<F, N>::cutoff() -> F      (biquad.rs:227-232)
//!   (F = f32 and f64: the prelude64 impls call them on the f64 nodes) Lowpole / Highpole / DCBlock ::<F, ..>::cutoff() -> F
//!   (filter.rs:20-130, :340-380)  Allpole::<F, N>::delay() -> F (filter.rs:270-296: store the delay beside `eta`)
//!   AllNest::coefficient() / inner() -> &X          (delay.rs:294-302)     Tap / TapLinear::delay_range() -> (f32, f32) (delay.rs:148-160,386)
//!   Dsf::spacing_roughness() -> (f32, f32)          (oscillator.rs:120)    Mls::bits() -> u32                        (noise.rs:101)
//!   Feedback::inner() / Feedback2::inner_pair()     (feedback.rs:71,183)   Reverb::time_diffusion_filter()           (reverb.rs:154-162)
//!   MultiBus / MultiStack / Reduce / MultiBranch / Chain ::nodes() -> &[X]  (audionode.rs:2065-2673)
//! Everything else goes through the public API (`Pipe::left()/right()`, `Constant::value()`, `Svf::cutoff()/q()/gain()`, `Biquad::coefs()`, `AudioNode::ID`, ...).
#![allow(clippy::missing_safety_doc)]
use crate::audionode::*;
use crate::audiounit::AudioUnit;
use crate::buffer::{BufferMut, BufferRef};
use crate::combinator::An;
use crate::math::AttoHash;
use crate::setting::{Address, Parameter, Setting};
use crate::signal::{Routing, SignalFrame};
use crate::system::System;
use crate::*;
use core::ffi::{c_char, c_int, c_void};
use numeric_array::typenum::*;
extern crate alloc;
use alloc::{string::String, vec::Vec};

#[repr(C)] pub struct FdspNode { _p: [u8; 0] }
#[repr(C)] pub struct FdspBank { _p: [u8; 0] }
#[repr(C)] pub struct FdspShared { _p: [u8; 0] }
#[repr(C)] pub struct FdspGroup { _p: [u8; 0] }

pub const FDSP_OUT_VOICES: u32 = 1;
pub const FDSP_OUT_MIX: u32 = 2;

#[link(name = "fundsp_b200")]
extern "C" {
    fn fdsp_last_error() -> *const c_char;
    fn fdsp_constant(n: c_int, values: *const f32) -> *mut FdspNode;
    fn fdsp_pass() -> *mut FdspNode;
    fn fdsp_multipass(n: c_int) -> *mut FdspNode;
    fn fdsp_sink(n: c_int) -> *mut FdspNode;
    fn fdsp_multisplit(m: c_int, n: c_int) -> *mut FdspNode;
    fn fdsp_multijoin(m: c_int, n: c_int) -> *mut FdspNode;
    fn fdsp_sine() -> *mut FdspNode;
    fn fdsp_wavesynth(table: c_int, outputs: c_int) -> *mut FdspNode;
    fn fdsp_noise() -> *mut FdspNode;
    fn fdsp_fixed_svf(mode: c_int, cutoff: f32, q: f32, gain: f32) -> *mut FdspNode;
    fn fdsp_moog(cutoff: f32, q: f32, inputs: c_int) -> *mut FdspNode;
    fn fdsp_fir(n: c_int, weights: *const f32) -> *mut FdspNode;
    fn fdsp_delay(seconds: f64) -> *mut FdspNode;
    fn fdsp_pan(value: f32) -> *mut FdspNode;
    fn fdsp_adsr_live(a: f32, d: f32, s: f32, r: f32) -> *mut FdspNode;
    fn fdsp_map(inputs: c_int, outputs: c_int, closure: *const c_char, ncaptures: c_int, names: *const *const c_char, values: *const f32) -> *mut FdspNode;
    fn fdsp_shape_fn(closure: *const c_char, ncaptures: c_int, names: *const *const c_char, values: *const f32) -> *mut FdspNode;
    fn fdsp_envelope_in(interval: f64, inputs: c_int, outputs: c_int, closure: *const c_char, ncaptures: c_int, names: *const *const c_char, values: *const f32) -> *mut FdspNode;
    fn fdsp_envelope_text(interval: f64, outputs: c_int, closure: *const c_char, ncaptures: c_int, names: *const *const c_char, values: *const f32) -> *mut FdspNode;
    fn fdsp_update(x: *mut FdspNode, dt: f32, closure: *const c_char, ncaptures: c_int, names: *const *const c_char, values: *const f32) -> *mut FdspNode;
    fn fdsp_convolve(response: *const f32, n: c_int) -> *mut FdspNode;
    fn fdsp_shaper(kind: c_int, p0: f32, p1: f32) -> *mut FdspNode;
    fn fdsp_shaper_adaptive(timescale: f64, inner_kind: c_int, p0: f32, p1: f32) -> *mut FdspNode;
    fn fdsp_nl_biquad(fb: c_int, mode: c_int, shape: c_int, p0: f32, p1: f32, inputs: c_int, center: f32, q: f32, gain: f32) -> *mut FdspNode;
    fn fdsp_nl_biquad_adaptive(fb: c_int, mode: c_int, timescale: f64, inner_kind: c_int, p0: f32, p1: f32, inputs: c_int, center: f32, q: f32, gain: f32) -> *mut FdspNode;
    fn fdsp_pipe(x: *mut FdspNode, y: *mut FdspNode) -> *mut FdspNode;
    fn fdsp_stack(x: *mut FdspNode, y: *mut FdspNode) -> *mut FdspNode;
    fn fdsp_branch(x: *mut FdspNode, y: *mut FdspNode) -> *mut FdspNode;
    fn fdsp_bus(x: *mut FdspNode, y: *mut FdspNode) -> *mut FdspNode;
    fn fdsp_thru(x: *mut FdspNode) -> *mut FdspNode;
    fn fdsp_binop(op: c_int, x: *mut FdspNode, y: *mut FdspNode) -> *mut FdspNode;
    fn fdsp_unop(kind: c_int, scalar: f32, x: *mut FdspNode) -> *mut FdspNode;
    fn fdsp_multi(kind: c_int, op: c_int, n: c_int, nodes: *const *mut FdspNode) -> *mut FdspNode;
    fn fdsp_feedback(x: *mut FdspNode, hadamard: c_int) -> *mut FdspNode;
    // the rest of SURVEY.md §8(a): routing, audio-rate filters, oscillators, delays, feedback forms, reverb, envelopes, Net
    fn fdsp_split(n: c_int) -> *mut FdspNode;
    fn fdsp_join(n: c_int) -> *mut FdspNode;
    fn fdsp_reverse(n: c_int) -> *mut FdspNode;
    fn fdsp_impulse(n: c_int) -> *mut FdspNode;
    fn fdsp_svf(mode: c_int, cutoff: f32, q: f32, gain: f32) -> *mut FdspNode;
    fn fdsp_sine_f64() -> *mut FdspNode;
    fn fdsp_fixed_svf_f64(mode: c_int, cutoff: f32, q: f32, gain: f32) -> *mut FdspNode;
    fn fdsp_svf_f64(mode: c_int, cutoff: f32, q: f32, gain: f32) -> *mut FdspNode;
    fn fdsp_biquad_f64(a1: f32, a2: f32, b0: f32, b1: f32, b2: f32) -> *mut FdspNode;
    fn fdsp_butterpass_f64(cutoff: f32, inputs: c_int) -> *mut FdspNode;
    fn fdsp_resonator_f64(center: f32, q: f32, inputs: c_int) -> *mut FdspNode;
    fn fdsp_onepole_f64(kind: c_int, param: f32, inputs: c_int) -> *mut FdspNode;
    fn fdsp_biquad(a1: f32, a2: f32, b0: f32, b1: f32, b2: f32) -> *mut FdspNode;
    fn fdsp_biquad_bank() -> *mut FdspNode;
    fn fdsp_butterpass(cutoff: f32, inputs: c_int) -> *mut FdspNode;
    fn fdsp_resonator(center: f32, q: f32, inputs: c_int) -> *mut FdspNode;
    fn fdsp_tick(n: c_int) -> *mut FdspNode;
    fn fdsp_allnest(coefficient: f32, x: *mut FdspNode, inputs: c_int) -> *mut FdspNode;
    fn fdsp_phase_osc(kind: c_int) -> *mut FdspNode;
    fn fdsp_dsf(inputs: c_int, harmonic_spacing: f32, roughness: f32) -> *mut FdspNode;
    fn fdsp_mls(bits: c_int) -> *mut FdspNode;
    fn fdsp_tap(taps: c_int, linear: c_int, min_delay: f32, max_delay: f32) -> *mut FdspNode;
    fn fdsp_feedback2(x: *mut FdspNode, y: *mut FdspNode, hadamard: c_int) -> *mut FdspNode;
    fn fdsp_feedback_unit(delay: f64, x: *mut FdspNode) -> *mut FdspNode;
    fn fdsp_reverb3(time: f64, diffusion: f64, filter: *mut FdspNode) -> *mut FdspNode;
    fn fdsp_panner() -> *mut FdspNode;
    fn fdsp_var(value: f32) -> *mut FdspNode;
    fn fdsp_shared_wrap(cell: *mut u32, release: Option<unsafe extern "C" fn(*mut c_void)>, user: *mut c_void) -> *mut FdspShared;
    fn fdsp_var_fn(s: *mut FdspShared, outputs: c_int, closure: *const c_char, ncaptures: c_int, names: *const *const c_char, values: *const f32) -> *mut FdspNode;
    fn fdsp_shared_free(s: *mut FdspShared);
    fn fdsp_var_shared(s: *mut FdspShared) -> *mut FdspNode;
    fn fdsp_monitor_shared(s: *mut FdspShared, kind: c_int, timescale: f64) -> *mut FdspNode;
    fn fdsp_timer(s: *mut FdspShared) -> *mut FdspNode;
    fn fdsp_net_new(inputs: c_int, outputs: c_int) -> *mut FdspNode;
    fn fdsp_net_push(net: *mut FdspNode, unit: *mut FdspNode) -> c_int;
    fn fdsp_net_connect(net: *mut FdspNode, source: c_int, source_port: c_int, target: c_int, target_port: c_int) -> c_int;
    fn fdsp_net_connect_input(net: *mut FdspNode, global_input: c_int, target: c_int, target_port: c_int) -> c_int;
    fn fdsp_net_connect_output(net: *mut FdspNode, source: c_int, source_port: c_int, global_output: c_int) -> c_int;
    fn fdsp_net_pass_through(net: *mut FdspNode, global_input: c_int, global_output: c_int) -> c_int;
    fn fdsp_bank_create_from_net(net: *mut FdspNode, device: c_int, out_mode: u32, out: *mut *mut FdspBank) -> c_int;
    fn fdsp_bank_voice_of_vertex(b: *const FdspBank, vertex: c_int) -> c_int;
    // live edits of a running bank (Net::replace / remove / crossfade, Slot::set, Sequencer::push / edit)
    fn fdsp_bank_replace_voice(b: *mut FdspBank, voice: u32, unit: *mut FdspNode) -> c_int;
    fn fdsp_bank_remove_voice(b: *mut FdspBank, voice: u32) -> c_int;
    fn fdsp_bank_crossfade_voice(b: *mut FdspBank, voice: u32, fade_ease: c_int, fade_time: f32, unit: *mut FdspNode) -> c_int;
    fn fdsp_slot(unit: *mut FdspNode) -> *mut FdspNode;
    fn fdsp_bank_slot_set(b: *mut FdspBank, voice: u32, fade_ease: c_int, fade_time: f64, unit: *mut FdspNode) -> c_int;
    fn fdsp_event(x: *mut FdspNode, start: f64, end: f64, fade_ease: c_int, fade_in: f64, fade_out: f64) -> *mut FdspNode;
    fn fdsp_event_loop(x: *mut FdspNode, start: f64, end: f64, fade_ease: c_int, fade_in: f64, fade_out: f64, loop_seconds: f64) -> *mut FdspNode;
    fn fdsp_bank_push_event(b: *mut FdspBank, event: *mut FdspNode, voice: *mut u32) -> c_int;
    fn fdsp_bank_edit_event(b: *mut FdspBank, voice: u32, end_time: f64, fade_out: f64) -> c_int;
    fn fdsp_bank_time(b: *const FdspBank) -> f64;
    fn fdsp_node_phase(n: *mut FdspNode, phase: f32) -> c_int;
    fn fdsp_node_seed(n: *mut FdspNode, seed: u64) -> c_int;
    fn fdsp_node_free(n: *mut FdspNode);
    fn fdsp_bank_create(voices: *const *mut FdspNode, n: u32, device: c_int, out_mode: u32, out: *mut *mut FdspBank) -> c_int;
    fn fdsp_bank_destroy(b: *mut FdspBank);
    fn fdsp_bank_clone(b: *const FdspBank, out: *mut *mut FdspBank) -> c_int;
    fn fdsp_bank_inputs(b: *const FdspBank) -> c_int;
    fn fdsp_bank_outputs(b: *const FdspBank) -> c_int;
    fn fdsp_bank_set_sample_rate(b: *mut FdspBank, sr: f64) -> c_int;
    fn fdsp_bank_reset(b: *mut FdspBank) -> c_int;
    fn fdsp_bank_allocate(b: *mut FdspBank, max_render_samples: u64) -> c_int;
    fn fdsp_bank_set(b: *mut FdspBank, voice: u32, kind: c_int, v: *const f32, nv: c_int, seed: u64, addr: *const i64, naddr: c_int) -> c_int;
    fn fdsp_bank_set_voices(b: *mut FdspBank, kind: c_int, voices: *const u32, n: u32, v: *const f32, nv: c_int, seeds: *const u64, addr: *const i64,
                            naddr: c_int, failed_entry: *mut u32) -> c_int;
    fn fdsp_bank_set_voices_device(b: *mut FdspBank, kind: c_int, voices: *const u32, n: u32, values_dev: *const f32, nv: c_int, addr: *const i64,
                                   naddr: c_int, stream: *mut c_void, failed_entry: *mut u32) -> c_int;
    fn fdsp_bank_process(b: *mut FdspBank, size: u32, input: *const f32, output: *mut f32) -> c_int;
    fn fdsp_bank_render(b: *mut FdspBank, n: u64, input: *const f32, out_voices: *mut f32, out_mix: *mut f32) -> c_int;
    // multi-GPU mix-down (csrc/host/group.h)
    fn fdsp_group_unique_id(id: *mut c_void, bytes: u64) -> c_int;
    fn fdsp_group_create(nranks: c_int, rank: c_int, id: *const c_void, device: c_int, out: *mut *mut FdspGroup) -> c_int;
    fn fdsp_group_destroy(g: *mut FdspGroup);
    fn fdsp_bank_render_reduced(b: *mut FdspBank, g: *mut FdspGroup, n: u64, input: *const f32, out_mix: *mut f32, root: c_int) -> c_int;
}

fn last_error() -> String {
    unsafe {
        let p = fdsp_last_error();
        if p.is_null() { return String::new(); }
        let mut n = 0usize;
        while *p.add(n) != 0 { n += 1; }
        String::from_utf8_lossy(core::slice::from_raw_parts(p as *const u8, n)).into_owned()
    }
}
fn check(rc: c_int) -> Result<(), String> { if rc == 0 { Ok(()) } else { Err(last_error()) } }

/// A typed graph lowers itself: one builder call per node, depth first, left to right — the order the reference constructs and pings
/// its nodes in (audionode.rs:156-161), so the deterministic phase hashes of the GPU voices equal the ones the Rust tree computed.
pub trait Lower { unsafe fn lower(&self) -> *mut FdspNode; }

impl<X: AudioNode + Lower> Lower for An<X> { unsafe fn lower(&self) -> *mut FdspNode { self.0.lower() } }

impl<X, Y> Lower for Pipe<X, Y> where X: AudioNode + Lower, Y: AudioNode<Inputs = X::Outputs> + Lower {
    unsafe fn lower(&self) -> *mut FdspNode { fdsp_pipe(self.left().lower(), self.right().lower()) }            // audionode.rs:1370
}
impl<X, Y> Lower for Stack<X, Y> where X: AudioNode + Lower, Y: AudioNode + Lower, X::Inputs: core::ops::Add<Y::Inputs>, X::Outputs: core::ops::Add<Y::Outputs>,
    <X::Inputs as core::ops::Add<Y::Inputs>>::Output: Size<f32>, <X::Outputs as core::ops::Add<Y::Outputs>>::Output: Size<f32> {
    unsafe fn lower(&self) -> *mut FdspNode { fdsp_stack(self.left().lower(), self.right().lower()) }           // audionode.rs:1494
}
impl<X, Y> Lower for Branch<X, Y> where X: AudioNode + Lower, Y: AudioNode<Inputs = X::Inputs> + Lower, X::Outputs: core::ops::Add<Y::Outputs>,
    <X::Outputs as core::ops::Add<Y::Outputs>>::Output: Size<f32> {
    unsafe fn lower(&self) -> *mut FdspNode { fdsp_branch(self.left().lower(), self.right().lower()) }          // audionode.rs:1651
}
impl<X, Y> Lower for Bus<X, Y> where X: AudioNode + Lower, Y: AudioNode<Inputs = X::Inputs, Outputs = X::Outputs> + Lower {
    unsafe fn lower(&self) -> *mut FdspNode { fdsp_bus(self.left().lower(), self.right().lower()) }             // audionode.rs:1794
}
impl<X: AudioNode + Lower> Lower for Thru<X> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_thru(self.inner().lower()) } }   // audionode.rs:1948

/// `+ - *` between graphs: Binop<FrameAdd|FrameSub|FrameMul, X, Y> (audionode.rs:850-1027); op 0 add, 1 sub, 2 mul.
pub trait BinopCode { const OP: c_int; }
impl<N: Size<f32>> BinopCode for FrameAdd<N> { const OP: c_int = 0; }
impl<N: Size<f32>> BinopCode for FrameSub<N> { const OP: c_int = 1; }
impl<N: Size<f32>> BinopCode for FrameMul<N> { const OP: c_int = 2; }
impl<B, X, Y> Lower for Binop<B, X, Y> where B: FrameBinop<X::Outputs> + BinopCode, X: AudioNode + Lower, Y: AudioNode<Outputs = X::Outputs> + Lower,
    X::Inputs: core::ops::Add<Y::Inputs>, <X::Inputs as core::ops::Add<Y::Inputs>>::Output: Size<f32> {
    unsafe fn lower(&self) -> *mut FdspNode { fdsp_binop(B::OP, self.left().lower(), self.right().lower()) }
}
/// `-x`, `x + s`, `s - x`, `x * s`: Unop (audionode.rs:1229-1326); kind 0 neg, 1 +s, 2 -x+s, 3 *s. Needs the `scalar()` accessors.
pub trait UnopCode { const KIND: c_int; fn scalar_value(&self) -> f32; }
impl<N: Size<f32>> UnopCode for FrameNeg<N> { const KIND: c_int = 0; fn scalar_value(&self) -> f32 { 0.0 } }
impl<N: Size<f32>> UnopCode for FrameAddScalar<N> { const KIND: c_int = 1; fn scalar_value(&self) -> f32 { self.scalar() } }
impl<N: Size<f32>> UnopCode for FrameNegAddScalar<N> { const KIND: c_int = 2; fn scalar_value(&self) -> f32 { self.scalar() } }
impl<N: Size<f32>> UnopCode for FrameMulScalar<N> { const KIND: c_int = 3; fn scalar_value(&self) -> f32 { self.scalar() } }
impl<X, U> Lower for Unop<X, U> where X: AudioNode + Lower, U: FrameUnop<X::Outputs> + UnopCode {
    unsafe fn lower(&self) -> *mut FdspNode { fdsp_unop(U::KIND, self.unop().scalar_value(), self.inner().lower()) }
}

impl<N: Size<f32>> Lower for Constant<N> {
    unsafe fn lower(&self) -> *mut FdspNode { let v = self.value(); fdsp_constant(N::I32, v.as_ptr()) }        // audionode.rs:465
}
impl Lower for Pass { unsafe fn lower(&self) -> *mut FdspNode { fdsp_pass() } }
/// A `Shape` as the C ABI names it: kind 0 Clip .. 6 Atan with its two parameters, or one of those inside `Adaptive` (timescale > 0).
/// Needs the `timescale()` / `inner()` accessors of Adaptive and `shape()` of Shaper.
pub trait ShapeCode { fn code(&self) -> (c_int, f32, f32, f64); }
impl ShapeCode for crate::shape::Clip { fn code(&self) -> (c_int, f32, f32, f64) { (0, self.0, 0.0, 0.0) } }
impl ShapeCode for crate::shape::ClipTo { fn code(&self) -> (c_int, f32, f32, f64) { (1, self.0, self.1, 0.0) } }
impl ShapeCode for crate::shape::Tanh { fn code(&self) -> (c_int, f32, f32, f64) { (2, self.0, 0.0, 0.0) } }
impl ShapeCode for crate::shape::Softsign { fn code(&self) -> (c_int, f32, f32, f64) { (3, self.0, 0.0, 0.0) } }
impl ShapeCode for crate::shape::Crush { fn code(&self) -> (c_int, f32, f32, f64) { (4, self.0, 0.0, 0.0) } }
impl ShapeCode for crate::shape::SoftCrush { fn code(&self) -> (c_int, f32, f32, f64) { (5, self.0, 0.0, 0.0) } }
impl ShapeCode for crate::shape::Atan { fn code(&self) -> (c_int, f32, f32, f64) { (6, self.0, 0.0, 0.0) } }
impl<S: crate::shape::Shape + ShapeCode> ShapeCode for crate::shape::Adaptive<S> {
    fn code(&self) -> (c_int, f32, f32, f64) {   // shape.rs:156-200; a nested Adaptive gives kind -1, which the C ABI refuses
        let (k, p0, p1, t) = self.inner().code();
        (if t > 0.0 { -1 } else { k }, p0, p1, self.timescale() as f64)
    }
}
impl<S: crate::shape::Shape + ShapeCode> Lower for crate::shape::Shaper<S> {
    unsafe fn lower(&self) -> *mut FdspNode {   // shape.rs:205-249
        let (k, p0, p1, t) = self.shape().code();
        if t > 0.0 { fdsp_shaper_adaptive(t, k, p0, p1) } else { fdsp_shaper(k, p0, p1) }
    }
}
/// The nonlinear biquads (biquad.rs:494-920) with a fixed (center, q[, gain]): `fb` 1 FixedFbBiquad, 0 FixedDirtyBiquad; `mode` 0
/// resonator, 1 lowpass, 2 highpass, 3 bell. Needs the `shape()` / `center()` / `q()` / `gain()` accessors.
pub unsafe fn lower_nl_biquad<S: ShapeCode>(fb: c_int, mode: c_int, shape: &S, center: f32, q: f32, gain: f32) -> *mut FdspNode {
    let (k, p0, p1, t) = shape.code();
    if t > 0.0 { fdsp_nl_biquad_adaptive(fb, mode, t, k, p0, p1, 1, center, q, gain) } else { fdsp_nl_biquad(fb, mode, k, p0, p1, 1, center, q, gain) }
}
impl<N: Size<f32>> Lower for MultiPass<N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_multipass(N::I32) } }
impl<N: Size<f32>> Lower for Sink<N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_sink(N::I32) } }
impl Lower for crate::oscillator::Sine<f32> {
    unsafe fn lower(&self) -> *mut FdspNode { let n = fdsp_sine(); if let Some(p) = self.initial_phase() { fdsp_node_phase(n, p); } n }   // `.phase(p)`
}
impl<N: Size<f32>> Lower for crate::wavetable::WaveSynth<N> {
    unsafe fn lower(&self) -> *mut FdspNode {
        // table_kind(): 0 saw, 1 square, 2 triangle, 3 organ, 4 soft saw, 5 hammond (the lazily built global tables of wavetable.rs:493-623)
        let n = fdsp_wavesynth(self.table_kind() as c_int, N::I32);
        if let Some(p) = self.initial_phase() { fdsp_node_phase(n, p); }
        n
    }
}
impl Lower for crate::noise::Noise {
    unsafe fn lower(&self) -> *mut FdspNode { let n = fdsp_noise(); if let Some(s) = self.seed() { fdsp_node_seed(n, s); } n }            // `.seed(s)`
}
/// SVF mode index: 0 lowpass 1 highpass 2 bandpass 3 notch 4 peak 5 allpass 6 bell 7 lowshelf 8 highshelf (svf.rs:26-221).
pub trait SvfModeIndex { const INDEX: c_int; }
impl SvfModeIndex for crate::svf::LowpassMode<f32> { const INDEX: c_int = 0; }
impl SvfModeIndex for crate::svf::HighpassMode<f32> { const INDEX: c_int = 1; }
impl SvfModeIndex for crate::svf::BandpassMode<f32> { const INDEX: c_int = 2; }
impl SvfModeIndex for crate::svf::NotchMode<f32> { const INDEX: c_int = 3; }
impl SvfModeIndex for crate::svf::PeakMode<f32> { const INDEX: c_int = 4; }
impl SvfModeIndex for crate::svf::AllpassMode<f32> { const INDEX: c_int = 5; }
impl SvfModeIndex for crate::svf::BellMode<f32> { const INDEX: c_int = 6; }
impl SvfModeIndex for crate::svf::LowshelfMode<f32> { const INDEX: c_int = 7; }
impl SvfModeIndex for crate::svf::HighshelfMode<f32> { const INDEX: c_int = 8; }
impl<M: crate::svf::SvfMode<f32> + SvfModeIndex> Lower for crate::svf::FixedSvf<f32, M> {
    unsafe fn lower(&self) -> *mut FdspNode { let p = self.params(); fdsp_fixed_svf(M::INDEX, p.cutoff, p.q, p.gain) }                   // svf.rs:857
}
impl<N: Size<f32>> Lower for crate::moog::Moog<f32, N> {
    unsafe fn lower(&self) -> *mut FdspNode { let (c, q) = self.cutoff_q(); fdsp_moog(c, q, N::I32) }                                    // moog.rs:11-46
}
impl<N: Size<f32>> Lower for crate::fir::Fir<N> {
    unsafe fn lower(&self) -> *mut FdspNode { let w = self.weights(); fdsp_fir(N::I32, w.as_ptr()) }                                     // fir.rs:11-41
}
impl Lower for crate::delay::Delay { unsafe fn lower(&self) -> *mut FdspNode { fdsp_delay(self.length_seconds()) } }                       // delay.rs:69
impl Lower for crate::pan::Panner<U1> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_pan(self.pan_value()) } }                           // pan.rs:19
impl Lower for crate::convolve::Convolver {
    unsafe fn lower(&self) -> *mut FdspNode { let h = self.response(); fdsp_convolve(h.as_ptr(), h.len() as c_int) }                     // convolve.rs:9
}
// ---- the rest of SURVEY.md §8(a). Type parameters as in v0.23.0; `F = f32` is the prelude32 instantiation the hot path uses.
impl<N: Size<f32>> Lower for Split<N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_split(N::I32) } }                               // audionode.rs:527
impl<N: Size<f32>> Lower for Join<N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_join(N::I32) } }                                 // audionode.rs:617
impl<M: Size<f32>, N: Size<f32>> Lower for MultiSplit<M, N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_multisplit(M::I32, N::I32) } }   // :571
impl<M: Size<f32>, N: Size<f32>> Lower for MultiJoin<M, N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_multijoin(M::I32, N::I32) } }     // :668
impl<N: Size<f32>> Lower for Reverse<N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_reverse(N::I32) } }                           // audionode.rs:2808
impl<N: Size<f32>> Lower for Impulse<N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_impulse(N::I32) } }                           // audionode.rs:2841
/// Svf<f32, M> with audio-rate cutoff / Q (/ gain) inputs (svf.rs:748): the initial parameters are public accessors.
impl<M: crate::svf::SvfMode<f32> + SvfModeIndex> Lower for crate::svf::Svf<f32, M> {
    unsafe fn lower(&self) -> *mut FdspNode { fdsp_svf(M::INDEX, self.cutoff(), self.q(), self.gain()) }
}
// prelude64 (F = f64): Sine<f64>, FixedSvf<f64, M>, Svf<f64, M>. Their f64 parameters were set from f32 values (F::from_f32), so
// `as f32` gives those values back exactly; the f64 state is built on the device (csrc/dsp/nodes.cuh Sine64, FixedSvf64, Svf64).
impl SvfModeIndex for crate::svf::LowpassMode<f64> { const INDEX: c_int = 0; }
impl SvfModeIndex for crate::svf::HighpassMode<f64> { const INDEX: c_int = 1; }
impl SvfModeIndex for crate::svf::BandpassMode<f64> { const INDEX: c_int = 2; }
impl SvfModeIndex for crate::svf::NotchMode<f64> { const INDEX: c_int = 3; }
impl SvfModeIndex for crate::svf::PeakMode<f64> { const INDEX: c_int = 4; }
impl SvfModeIndex for crate::svf::AllpassMode<f64> { const INDEX: c_int = 5; }
impl SvfModeIndex for crate::svf::BellMode<f64> { const INDEX: c_int = 6; }
impl SvfModeIndex for crate::svf::LowshelfMode<f64> { const INDEX: c_int = 7; }
impl SvfModeIndex for crate::svf::HighshelfMode<f64> { const INDEX: c_int = 8; }
impl Lower for crate::oscillator::Sine<f64> {
    unsafe fn lower(&self) -> *mut FdspNode { let n = fdsp_sine_f64(); if let Some(p) = self.initial_phase() { fdsp_node_phase(n, p as f32); } n }
}
impl<M: crate::svf::SvfMode<f64> + SvfModeIndex> Lower for crate::svf::FixedSvf<f64, M> {
    unsafe fn lower(&self) -> *mut FdspNode { let p = self.params(); fdsp_fixed_svf_f64(M::INDEX, p.cutoff as f32, p.q as f32, p.gain as f32) }
}
impl<M: crate::svf::SvfMode<f64> + SvfModeIndex> Lower for crate::svf::Svf<f64, M> {
    unsafe fn lower(&self) -> *mut FdspNode { fdsp_svf_f64(M::INDEX, self.cutoff() as f32, self.q() as f32, self.gain() as f32) }
}
impl Lower for crate::biquad::Biquad<f32> {
    unsafe fn lower(&self) -> *mut FdspNode { let c = self.coefs(); fdsp_biquad(c.a1, c.a2, c.b0, c.b1, c.b2) }                        // biquad.rs:136-165
}
impl Lower for crate::biquad_bank::BiquadBank<wide::f32x8> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_biquad_bank() } }          // biquad_bank.rs:14; lanes are set with Setting::biquad(..).index(l)
impl<N: Size<f32>> Lower for crate::biquad::ButterLowpass<f32, N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_butterpass(self.cutoff(), N::I32) } }   // N = U1 fixed, U2 audio-rate cutoff
impl<N: Size<f32>> Lower for crate::biquad::Resonator<f32, N> {
    unsafe fn lower(&self) -> *mut FdspNode { let (c, q) = self.center_q(); fdsp_resonator(c, q, N::I32) }                              // N = U1 fixed, U3 audio-rate center / Q
}
// prelude64 biquads and one-poles (F = f64): their parameters came from f32 values (F::from_f32), so `as f32` is exact. Biquad<f64>'s
// coefficients are f64 values set from f32 settings or by BiquadCoefs::<f64> formulas; only the former round-trip through f32.
impl Lower for crate::biquad::Biquad<f64> {
    unsafe fn lower(&self) -> *mut FdspNode { let c = self.coefs(); fdsp_biquad_f64(c.a1 as f32, c.a2 as f32, c.b0 as f32, c.b1 as f32, c.b2 as f32) }
}
impl<N: Size<f32>> Lower for crate::biquad::ButterLowpass<f64, N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_butterpass_f64(self.cutoff() as f32, N::I32) } }
impl<N: Size<f32>> Lower for crate::biquad::Resonator<f64, N> {
    unsafe fn lower(&self) -> *mut FdspNode { let (c, q) = self.center_q(); fdsp_resonator_f64(c as f32, q as f32, N::I32) }
}
impl<N: Size<f32>> Lower for crate::filter::Lowpole<f64, N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_onepole_f64(0, self.cutoff() as f32, N::I32) } }
impl<N: Size<f32>> Lower for crate::filter::Highpole<f64, N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_onepole_f64(1, self.cutoff() as f32, N::I32) } }
impl<N: Size<f32>> Lower for crate::filter::Allpole<f64, N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_onepole_f64(2, self.delay() as f32, N::I32) } }
impl Lower for crate::filter::DCBlock<f64> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_onepole_f64(3, self.cutoff() as f32, 1) } }
impl Lower for crate::filter::Pinkpass<f64> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_onepole_f64(4, 0.0, 1) } }
impl<N: Size<f32>> Lower for crate::delay::Tick<N> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_tick(N::I32) } }                    // delay.rs:19
impl<N: Size<f32>, X: AudioNode<Inputs = U1, Outputs = U1> + Lower> Lower for crate::delay::AllNest<N, X> {
    unsafe fn lower(&self) -> *mut FdspNode { fdsp_allnest(self.coefficient(), self.inner().lower(), N::I32) }                          // delay.rs:294 (N = U2: audio-rate coefficient)
}
impl<N> Lower for crate::delay::Tap<N> where N: Size<f32> + core::ops::Add<U1>, <N as core::ops::Add<U1>>::Output: Size<f32> {
    unsafe fn lower(&self) -> *mut FdspNode { let (lo, hi) = self.delay_range(); fdsp_tap(N::I32, 0, lo, hi) }                          // delay.rs:148 (cubic taps)
}
impl<N> Lower for crate::delay::TapLinear<N> where N: Size<f32> + core::ops::Add<U1>, <N as core::ops::Add<U1>>::Output: Size<f32> {
    unsafe fn lower(&self) -> *mut FdspNode { let (lo, hi) = self.delay_range(); fdsp_tap(N::I32, 1, lo, hi) }                          // delay.rs:386
}
impl Lower for crate::oscillator::Ramp<f32> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_phase_osc(0) } }                           // oscillator.rs:441
impl Lower for crate::oscillator::PolySaw<f32> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_phase_osc(1) } }                        // :529
impl Lower for crate::oscillator::PolySquare<f32> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_phase_osc(2) } }                     // :605
impl Lower for crate::oscillator::PolyPulse<f32> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_phase_osc(3) } }                      // :688
impl<N: Size<f32>> Lower for crate::oscillator::Dsf<N> {
    unsafe fn lower(&self) -> *mut FdspNode { let (h, r) = self.spacing_roughness(); fdsp_dsf(N::I32, h, r) }                           // oscillator.rs:120 (N = U1 fixed, U2 audio-rate roughness)
}
impl Lower for crate::noise::Mls { unsafe fn lower(&self) -> *mut FdspNode { fdsp_mls(self.bits() as c_int) } }                          // noise.rs:101
impl Lower for crate::pan::Panner<U2> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_panner() } }                                     // pan.rs:19 (audio-rate pan)
/// Feedback<N, X, FrameId | FrameHadamard> (feedback.rs:71) and Feedback2 (:183): the frame operator is a type, the C ABI takes a flag.
pub trait FeedbackFrame { const HADAMARD: c_int; }
impl<N: Size<f32>> FeedbackFrame for FrameId<N> { const HADAMARD: c_int = 0; }
impl<N: Size<f32>> FeedbackFrame for crate::feedback::FrameHadamard<N> { const HADAMARD: c_int = 1; }
impl<N, X, U> Lower for crate::feedback::Feedback<N, X, U> where N: Size<f32>, X: AudioNode<Inputs = N, Outputs = N> + Lower, U: FrameUnop<N> + FeedbackFrame {
    unsafe fn lower(&self) -> *mut FdspNode { fdsp_feedback(self.inner().lower(), U::HADAMARD) }
}
impl<N, X, Y, U> Lower for crate::feedback::Feedback2<N, X, Y, U>
where N: Size<f32>, X: AudioNode<Inputs = N, Outputs = N> + Lower, Y: AudioNode<Inputs = N, Outputs = N> + Lower, U: FrameUnop<N> + FeedbackFrame {
    unsafe fn lower(&self) -> *mut FdspNode { let (x, y) = self.inner_pair(); fdsp_feedback2(x.lower(), y.lower(), U::HADAMARD) }
}
impl<F: AudioNode<Inputs = U1, Outputs = U1> + Lower> Lower for crate::reverb::Reverb<F> {
    unsafe fn lower(&self) -> *mut FdspNode { let (t, d, f) = self.time_diffusion_filter(); fdsp_reverb3(t, d, f.lower()) }               // reverb.rs:154 (reverb3_stereo)
}
/// Shared controls over the application's own cell: the AtomicU32 behind `Shared` (`Shared::get_shared`, the only public way to it in
/// shared.rs) is wrapped, so `Shared::set` reaches the bank between calls and the bank's monitor / timer stores reach `Shared::value`.
/// The reference keeps the Arc of Var, VarFn, Monitor and Timer private: these need one accessor each (`shared_arc()`). The wrapper
/// holds an Arc clone of its own (leaked into `user`, dropped by `release_cell` when the library lets go of the cell's last reference),
/// so the memory outlives every node and bank that uses it even when the application drops its Shared and graph first.
unsafe extern "C" fn release_cell(user: *mut c_void) { drop(alloc::sync::Arc::from_raw(user as *const core::sync::atomic::AtomicU32)); }
unsafe fn wrap_cell(a: &alloc::sync::Arc<core::sync::atomic::AtomicU32>) -> *mut FdspShared {
    let keep = alloc::sync::Arc::into_raw(alloc::sync::Arc::clone(a)) as *mut c_void;
    fdsp_shared_wrap(a.as_ptr(), Some(release_cell), keep)
}
impl Lower for crate::shared::Var {                                                                                                       // shared.rs:84-131, ID 68
    unsafe fn lower(&self) -> *mut FdspNode { let s = wrap_cell(self.shared_arc()); let n = fdsp_var_shared(s); fdsp_shared_free(s); n }
}
impl Lower for crate::dynamics::Monitor {                                                                                                   // dynamics.rs:441-520, ID 56
    unsafe fn lower(&self) -> *mut FdspNode {
        let (kind, t) = match self.meter() { crate::dynamics::Meter::Sample => (0, 0.0), crate::dynamics::Meter::Peak(t) => (1, t), crate::dynamics::Meter::Rms(t) => (2, t) };
        let s = wrap_cell(self.shared_arc()); let n = fdsp_monitor_shared(s, kind, t); fdsp_shared_free(s); n
    }
}
impl Lower for crate::shared::Timer { unsafe fn lower(&self) -> *mut FdspNode { let s = wrap_cell(self.shared_arc()); let n = fdsp_timer(s); fdsp_shared_free(s); n } }   // shared.rs:203-250, ID 57
/// The N-ary combinators hold their units in a Frame<X, N> (audionode.rs:2065-2673); kind codes are the nodes' IDs.
macro_rules! lower_multi { ($t:ident, $kind:expr, $op:expr) => {
    impl<N: Size<f32> + Size<X>, X: AudioNode + Lower> Lower for $t<N, X> {
        unsafe fn lower(&self) -> *mut FdspNode { let hs: Vec<*mut FdspNode> = self.nodes().iter().map(|x| x.lower()).collect(); fdsp_multi($kind, $op, hs.len() as c_int, hs.as_ptr()) }
    }
} }
lower_multi!(MultiBus, 28, 0); lower_multi!(MultiStack, 30, 0); lower_multi!(MultiBranch, 33, 0); lower_multi!(Chain, 32, 0);
impl<N: Size<f32> + Size<X>, X: AudioNode + Lower, B: FrameBinop<X::Outputs> + BinopCode> Lower for Reduce<N, X, B> {
    unsafe fn lower(&self) -> *mut FdspNode { let hs: Vec<*mut FdspNode> = self.nodes().iter().map(|x| x.lower()).collect(); fdsp_multi(31, B::OP, hs.len() as c_int, hs.as_ptr()) }
}

/// `adsr_live(a, d, s, r)` is `EnvelopeIn` with the closure of adsr.rs:21-70: closures do not cross a C ABI, the closed form does.
pub struct AdsrLive { pub attack: f32, pub decay: f32, pub sustain: f32, pub release: f32 }
impl Lower for AdsrLive { unsafe fn lower(&self) -> *mut FdspNode { fdsp_adsr_live(self.attack, self.decay, self.sustain, self.release) } }

/// A closure of the signal that can also run on the GPU: the reference's node `X` (what runs on the CPU) plus the closure's text and
/// captured values, which `Lower` hands to `fdsp_map` / `fdsp_shape_fn` / `fdsp_envelope_in` / `fdsp_envelope_text`. Made by `gpu_map!`,
/// `gpu_shape_fn!`, `gpu_envelope_in!`, `gpu_envelope!` and `gpu_lfo!`, which take the closure ONCE: it is compiled by rustc for the CPU node and `stringify!`-ed for the GPU node, so
/// the two cannot drift apart. The text must stay inside the closure language of DESIGN.md §2 (f32 literals, the listed functions);
/// `fdsp_*` refuses anything else with the token and its column, and `GpuBank::new` returns that error.
#[derive(Clone)]
pub struct GpuClosure<X> { pub node: X, pub kind: c_int, pub interval: f64, pub text: &'static str, pub names: Vec<&'static str>, pub values: Vec<f32> }
impl<X: AudioNode> AudioNode for GpuClosure<X> {
    const ID: u64 = X::ID;
    type Inputs = X::Inputs;
    type Outputs = X::Outputs;
    fn reset(&mut self) { self.node.reset() }
    fn set_sample_rate(&mut self, sample_rate: f64) { self.node.set_sample_rate(sample_rate) }
    fn tick(&mut self, input: &Frame<f32, Self::Inputs>) -> Frame<f32, Self::Outputs> { self.node.tick(input) }
    fn process(&mut self, size: usize, input: &BufferRef, output: &mut BufferMut) { self.node.process(size, input, output) }
    fn set(&mut self, setting: Setting) { if let Parameter::Interval(t) = setting.parameter() { self.interval = *t as f64; } self.node.set(setting) }
    fn set_hash(&mut self, hash: u64) { self.node.set_hash(hash) }
    fn route(&mut self, input: &SignalFrame, frequency: f64) -> SignalFrame { self.node.route(input, frequency) }
}
impl<X: AudioNode> Lower for GpuClosure<X> {
    unsafe fn lower(&self) -> *mut FdspNode {
        let text: Vec<u8> = self.text.bytes().chain(core::iter::once(0)).collect();
        let names: Vec<Vec<u8>> = self.names.iter().map(|n| n.bytes().chain(core::iter::once(0)).collect()).collect();
        let ptrs: Vec<*const c_char> = names.iter().map(|n| n.as_ptr() as *const c_char).collect();
        let (i, o, nc) = (X::Inputs::I32, X::Outputs::I32, self.values.len() as c_int);
        let t = text.as_ptr() as *const c_char;
        match self.kind {
            0 => fdsp_map(i, o, t, nc, ptrs.as_ptr(), self.values.as_ptr()),
            1 => fdsp_shape_fn(t, nc, ptrs.as_ptr(), self.values.as_ptr()),
            4 => fdsp_envelope_text(self.interval, o, t, nc, ptrs.as_ptr(), self.values.as_ptr()),
            _ => fdsp_envelope_in(self.interval, i, o, t, nc, ptrs.as_ptr(), self.values.as_ptr()),
        }
    }
}
/// `gpu_map!(U1, U1, [drive], |x: &Frame<f32, U1>| tanh(x[0] * drive))`: `map(..)` (prelude.rs:1126) that lowers to `fdsp_map`.
/// The bracket lists the captured f32 variables.
#[macro_export]
macro_rules! gpu_map {
    ($i:ty, $o:ty, [$($c:ident),*], $($f:tt)+) => {
        $crate::combinator::An($crate::gpu::GpuClosure {
            node: $crate::audionode::Map::<_, $i, $o>::new($($f)+, $crate::signal::Routing::Arbitrary(0.0)),
            kind: 0, interval: 0.0, text: stringify!($($f)+), names: vec![$(stringify!($c)),*], values: vec![$($c as f32),*],
        })
    };
}
/// `gpu_var_fn!(&s, [g], |x: f32| (x * g, -x))`: `var_fn(&s, f)` (shared.rs:134-200, ID 70) that lowers to `fdsp_var_fn` over the
/// Shared's own cell; the output count is the closure's return type.
#[macro_export]
macro_rules! gpu_var_fn {
    ($s:expr, [$($c:ident),*], $($f:tt)+) => {
        $crate::combinator::An($crate::gpu::GpuVarFn {
            node: $crate::shared::VarFn::new($s, $($f)+), cell: ::alloc::sync::Arc::clone($s.get_shared()),
            text: stringify!($($f)+), names: vec![$(stringify!($c)),*], values: vec![$($c as f32),*],
        })
    };
}
/// `gpu_shape_fn!([h], |x: f32| tanh(x * h))`: `shape_fn(..)` (prelude.rs:1181) that lowers to `fdsp_shape_fn`.
#[macro_export]
macro_rules! gpu_shape_fn {
    ([$($c:ident),*], $($f:tt)+) => {
        $crate::combinator::An($crate::gpu::GpuClosure {
            node: $crate::shape::Shaper::new($crate::shape::ShapeFn($($f)+)),
            kind: 1, interval: 0.0, text: stringify!($($f)+), names: vec![$(stringify!($c)),*], values: vec![$($c as f32),*],
        })
    };
}
/// `gpu_envelope_in!(U2, [k], |t: f32, i: &Frame<f32, U2>| i[0] * k + t)`: `envelope_in(..)` (prelude32.rs:716, interval 2 ms) that lowers to
/// `fdsp_envelope_in`; the output count is the closure's return type. envelope2 / envelope3 are this with `|t, x| ..` / `|t, x, y| ..`
/// written over `i[0]` / `i[1]` (prelude32.rs:625-708).
#[macro_export]
macro_rules! gpu_envelope_in {
    ($i:ty, [$($c:ident),*], $($f:tt)+) => {
        $crate::combinator::An($crate::gpu::GpuClosure {
            node: $crate::envelope::EnvelopeIn::<f32, _, $i, _>::new(0.002, $($f)+),
            kind: 2, interval: 0.002f32 as f64, text: stringify!($($f)+), names: vec![$(stringify!($c)),*], values: vec![$($c as f32),*],
        })
    };
}
/// `gpu_envelope!([rate], |t: f32| 1000.0 + 500.0 * sin_hz(rate, t))`: `envelope(..)` (prelude32.rs:581, Envelope<f32> ID 14, interval
/// 2 ms) that lowers to `fdsp_envelope_text`: the GPU evaluates the closure at every sample point, with no horizon. The output count is
/// the closure's return type.
#[macro_export]
macro_rules! gpu_envelope {
    ([$($c:ident),*], $($f:tt)+) => {
        $crate::combinator::An($crate::gpu::GpuClosure {
            node: $crate::envelope::Envelope::<f32, _, _>::new(0.002, $($f)+),
            kind: 4, interval: 0.002f32 as f64, text: stringify!($($f)+), names: vec![$(stringify!($c)),*], values: vec![$($c as f32),*],
        })
    };
}
/// `gpu_lfo!(..)`: `lfo(..)` is `envelope(..)` (prelude32.rs:604).
#[macro_export]
macro_rules! gpu_lfo {
    ($($t:tt)+) => { $crate::gpu_envelope!($($t)+) };
}

/// `update(x, dt, f)` (system.rs, System ID 67) that can also run on the GPU: the reference's System (what runs on the CPU), a copy of x
/// that settings reach too (what is lowered) and the update function's text. Made by `gpu_update!`.
#[derive(Clone)]
pub struct GpuSystem<X: AudioNode, F: FnMut(f32, f32, &mut X) + Clone + Send + Sync> {
    pub node: System<X, F>, pub x: X, pub dt: f32, pub text: &'static str, pub names: Vec<&'static str>, pub values: Vec<f32>,
}
impl<X: AudioNode, F: FnMut(f32, f32, &mut X) + Clone + Send + Sync> AudioNode for GpuSystem<X, F> {
    const ID: u64 = 67;
    type Inputs = X::Inputs;
    type Outputs = X::Outputs;
    fn reset(&mut self) { self.node.reset() }
    fn set_sample_rate(&mut self, sample_rate: f64) { self.node.set_sample_rate(sample_rate); self.x.set_sample_rate(sample_rate) }
    fn tick(&mut self, input: &Frame<f32, Self::Inputs>) -> Frame<f32, Self::Outputs> { self.node.tick(input) }
    fn process(&mut self, size: usize, input: &BufferRef, output: &mut BufferMut) { self.node.process(size, input, output) }
    fn set(&mut self, setting: Setting) { self.x.set(setting.clone()); self.node.set(setting) }
    fn ping(&mut self, probe: bool, hash: AttoHash) -> AttoHash { self.node.ping(probe, hash) }
    fn route(&mut self, input: &SignalFrame, frequency: f64) -> SignalFrame { self.node.route(input, frequency) }
}
impl<X: AudioNode + Lower, F: FnMut(f32, f32, &mut X) + Clone + Send + Sync> Lower for GpuSystem<X, F> {
    unsafe fn lower(&self) -> *mut FdspNode {
        let text: Vec<u8> = self.text.bytes().chain(core::iter::once(0)).collect();
        let names: Vec<Vec<u8>> = self.names.iter().map(|n| n.bytes().chain(core::iter::once(0)).collect()).collect();
        let ptrs: Vec<*const c_char> = names.iter().map(|n| n.as_ptr() as *const c_char).collect();
        fdsp_update(self.x.lower(), self.dt, text.as_ptr() as *const c_char, self.values.len() as c_int, ptrs.as_ptr(), self.values.as_ptr())
    }
}
/// `gpu_update!(x, dt, [r], |t: f32, dt: f32, x: &mut _| x.set(Setting::center(600.0 + 400.0 * sin_hz(r, t)).right()))`: `update(x, dt, f)`
/// (prelude.rs, System ID 67) that lowers to `fdsp_update`. The body is `let`s and unconditional `x.set(Setting::..)` statements
/// (DESIGN.md §2); the GPU runs it at the same update points.
#[macro_export]
macro_rules! gpu_update {
    ($x:expr, $dt:expr, [$($c:ident),*], $($f:tt)+) => {{
        let x = $x;
        $crate::combinator::An($crate::gpu::GpuSystem {
            node: $crate::system::System::new(x.clone(), $dt, $($f)+), x: x.0, dt: $dt,
            text: stringify!($($f)+), names: vec![$(stringify!($c)),*], values: vec![$($c as f32),*],
        })
    }};
}

/// V voices of typed graphs evaluated in lockstep on one GPU; to the host ONE `AudioUnit` (audiounit.rs:21-95).
pub struct GpuBank { h: *mut FdspBank, inputs: usize, outputs: usize, failed: bool }
unsafe impl Send for GpuBank {}
unsafe impl Sync for GpuBank {}

impl GpuBank {
    /// `voices`: per-voice graphs (they may fall into several structural classes); `mix`: outputs() = channels of the summed voices,
    /// else V * channels per-voice outputs.
    pub fn new<X: AudioNode + Lower>(voices: &[An<X>], device: i32, mix: bool) -> Result<Self, String> {
        let mut hs: Vec<*mut FdspNode> = Vec::with_capacity(voices.len());
        for v in voices {
            let h = unsafe { v.lower() };
            if h.is_null() { for x in hs { unsafe { fdsp_node_free(x) } } return Err(last_error()); }
            hs.push(h);
        }
        let mut b: *mut FdspBank = core::ptr::null_mut();
        check(unsafe { fdsp_bank_create(hs.as_ptr(), hs.len() as u32, device, if mix { FDSP_OUT_MIX } else { FDSP_OUT_VOICES }, &mut b) })?;   // consumes the handles
        let (i, o) = unsafe { (fdsp_bank_inputs(b) as usize, fdsp_bank_outputs(b) as usize) };
        Ok(GpuBank { h: b, inputs: i, outputs: o, failed: false })
    }
    /// `Wave::render` for many blocks in one call (wave.rs:441-466): `out` is [outputs()][samples], channel-major.
    pub fn render(&mut self, samples: usize, input: Option<&[f32]>, out: &mut [f32]) -> Result<(), String> {
        assert!(out.len() >= self.outputs * samples);
        check(unsafe { fdsp_bank_render(self.h, samples as u64, input.map_or(core::ptr::null(), |x| x.as_ptr()), core::ptr::null_mut(), out.as_mut_ptr()) })
    }
    pub fn failed(&self) -> bool { self.failed }
}
/// Live edits keep the reference's names (INTEGRATION.md "A dynamic Net", "A Sequencer as one bank"); `voice` = `voice_of_vertex(NodeId)` for banks made from a Net.
impl GpuBank {
    /// A voice-separable `Net` handed over vertex by vertex (`NetBuilder` below) becomes a bank that mixes in the Net's own order.
    pub unsafe fn from_net_handle(net: *mut FdspNode, device: i32, mix: bool) -> Result<Self, String> {
        let mut b: *mut FdspBank = core::ptr::null_mut();
        check(fdsp_bank_create_from_net(net, device, if mix { FDSP_OUT_MIX } else { FDSP_OUT_VOICES }, &mut b))?;
        Ok(GpuBank { h: b, inputs: fdsp_bank_inputs(b) as usize, outputs: fdsp_bank_outputs(b) as usize, failed: false })
    }
    /// `AudioUnit::set` on many voices in one call: entry j sets voice `voices[j]` (j when `voices` is None) to
    /// `values[j * nvalues..(j + 1) * nvalues]` with Parameter index `kind` and the (type, value) address pairs of `fdsp_node_set`. The same
    /// as one `set` per entry in order; on a refusal, Err holds the refused entry's index (the entries before it are applied, the rest not).
    pub fn set_voices(&mut self, kind: i32, values: &[f32], nvalues: usize, voices: Option<&[u32]>, address: &[(i32, i64)]) -> Result<(), (u32, String)> {
        let n = match voices { Some(v) => v.len(), None => if nvalues > 0 { values.len() / nvalues } else { 0 } };
        if nvalues > 5 || values.len() < n * nvalues { return Err((0, String::from("set_voices: values holds fewer than n * nvalues values"))); }
        let addr: Vec<i64> = address.iter().flat_map(|&(t, v)| [t as i64, v]).collect();
        let mut failed = 0u32;
        let rc = unsafe {
            fdsp_bank_set_voices(self.h, kind as c_int, voices.map_or(core::ptr::null(), |v| v.as_ptr()), n as u32, values.as_ptr(), nvalues as c_int,
                                 core::ptr::null(), addr.as_ptr(), address.len() as c_int, &mut failed)
        };
        check(rc).map_err(|e| (failed, e))
    }
    /// `set_voices` with the values in device memory, their coefficients computed on the device (`fdsp_bank_set_voices_device`): `n` rows
    /// of `nvalues` f32 at `values_dev` on the bank's device, written on the CUDA stream `stream` (null: the legacy default stream). The
    /// call is asynchronous and orders itself after `stream`, and `stream` after it. On a refusal no entry is applied; Err holds the first
    /// refused entry's index.
    ///
    /// # Safety
    /// `values_dev` must point to `n * nvalues` floats of device memory that stay valid until `stream` has passed this call.
    pub unsafe fn set_voices_device(&mut self, kind: i32, values_dev: *const f32, n: u32, nvalues: usize, voices: Option<&[u32]>, address: &[(i32, i64)],
                                    stream: *mut c_void) -> Result<(), (u32, String)> {
        if nvalues > 5 || voices.map_or(false, |v| v.len() != n as usize) { return Err((0, String::from("set_voices_device: nvalues <= 5 and one voice per entry"))); }
        let addr: Vec<i64> = address.iter().flat_map(|&(t, v)| [t as i64, v]).collect();
        let mut failed = 0u32;
        let rc = fdsp_bank_set_voices_device(self.h, kind as c_int, voices.map_or(core::ptr::null(), |v| v.as_ptr()), n, values_dev, nvalues as c_int,
                                             addr.as_ptr(), address.len() as c_int, stream, &mut failed);
        check(rc).map_err(|e| (failed, e))
    }
    pub fn voice_of_vertex(&self, vertex: usize) -> Option<u32> { let v = unsafe { fdsp_bank_voice_of_vertex(self.h, vertex as c_int) }; if v < 0 { None } else { Some(v as u32) } }
    pub fn replace<X: AudioNode + Lower>(&mut self, voice: u32, unit: &An<X>) -> Result<(), String> { check(unsafe { fdsp_bank_replace_voice(self.h, voice, unit.lower()) }) }   // Net::replace (net.rs:460)
    pub fn remove(&mut self, voice: u32) -> Result<(), String> { check(unsafe { fdsp_bank_remove_voice(self.h, voice) }) }                                                       // Net::remove (net.rs:351)
    pub fn crossfade<X: AudioNode + Lower>(&mut self, voice: u32, fade: crate::sequencer::Fade, fade_time: f32, unit: &An<X>) -> Result<(), String> {                             // Net::crossfade (net.rs:480)
        check(unsafe { fdsp_bank_crossfade_voice(self.h, voice, fade as c_int, fade_time, unit.lower()) })
    }
    pub fn slot_set<X: AudioNode + Lower>(&mut self, voice: u32, fade: crate::sequencer::Fade, fade_time: f64, unit: &An<X>) -> Result<(), String> {                              // Slot::set (slot.rs:64)
        check(unsafe { fdsp_bank_slot_set(self.h, voice, fade as c_int, fade_time, unit.lower()) })
    }
    pub fn time(&self) -> f64 { unsafe { fdsp_bank_time(self.h) } }
}
/// `Slot::new(unit)` as a voice graph (slot.rs:33): lower the unit, wrap the handle.
pub struct SlotVoice<X>(pub An<X>);
impl<X: AudioNode + Lower> Lower for SlotVoice<X> { unsafe fn lower(&self) -> *mut FdspNode { fdsp_slot(self.0.lower()) } }
/// One Sequencer event as a voice (sequencer.rs:319-345); `loop_seconds` > 0 for a ReplayMode::Loop sequencer.
pub struct EventVoice<X> { pub unit: An<X>, pub start: f64, pub end: f64, pub fade: crate::sequencer::Fade, pub fade_in: f64, pub fade_out: f64, pub loop_seconds: f64 }
impl<X: AudioNode + Lower> Lower for EventVoice<X> {
    unsafe fn lower(&self) -> *mut FdspNode {
        if self.loop_seconds > 0.0 { fdsp_event_loop(self.unit.lower(), self.start, self.end, self.fade.clone() as c_int, self.fade_in, self.fade_out, self.loop_seconds) }
        else { fdsp_event(self.unit.lower(), self.start, self.end, self.fade.clone() as c_int, self.fade_in, self.fade_out) }
    }
}
/// Mirror of the Net construction calls (net.rs:204-213,320-345,520-640): vertex ids are the indices `Net::push` hands out.
pub struct NetBuilder { h: *mut FdspNode }
impl NetBuilder {
    pub fn new(inputs: usize, outputs: usize) -> Self { NetBuilder { h: unsafe { fdsp_net_new(inputs as c_int, outputs as c_int) } } }
    pub fn push<X: AudioNode + Lower>(&mut self, unit: &An<X>) -> Result<usize, String> { let v = unsafe { fdsp_net_push(self.h, unit.lower()) }; if v < 0 { Err(last_error()) } else { Ok(v as usize) } }
    pub fn connect(&mut self, source: usize, source_port: usize, target: usize, target_port: usize) -> Result<(), String> { check(unsafe { fdsp_net_connect(self.h, source as c_int, source_port as c_int, target as c_int, target_port as c_int) }) }
    pub fn connect_input(&mut self, global_input: usize, target: usize, target_port: usize) -> Result<(), String> { check(unsafe { fdsp_net_connect_input(self.h, global_input as c_int, target as c_int, target_port as c_int) }) }
    pub fn connect_output(&mut self, source: usize, source_port: usize, global_output: usize) -> Result<(), String> { check(unsafe { fdsp_net_connect_output(self.h, source as c_int, source_port as c_int, global_output as c_int) }) }
    pub fn pass_through(&mut self, global_input: usize, global_output: usize) -> Result<(), String> { check(unsafe { fdsp_net_pass_through(self.h, global_input as c_int, global_output as c_int) }) }
    /// The finished Net as a bank (consumes the handle) ...
    pub fn into_bank(self, device: i32, mix: bool) -> Result<GpuBank, String> { let h = self.h; core::mem::forget(self); unsafe { GpuBank::from_net_handle(h, device, mix) } }
    /// ... or as a node of a larger voice expression: any acyclic Net lowers to one fused program.
    pub fn into_node(self) -> NetNode { let h = self.h; core::mem::forget(self); NetNode(h) }
}
impl Drop for NetBuilder { fn drop(&mut self) { if !self.h.is_null() { unsafe { fdsp_node_free(self.h) } } } }
pub struct NetNode(*mut FdspNode);

impl AudioUnit for GpuBank {
    fn inputs(&self) -> usize { self.inputs }
    fn outputs(&self) -> usize { self.outputs }
    fn reset(&mut self) { if unsafe { fdsp_bank_reset(self.h) } != 0 { self.failed = true; } }
    fn set_sample_rate(&mut self, sr: f64) { if unsafe { fdsp_bank_set_sample_rate(self.h, sr) } != 0 { self.failed = true; } }
    fn allocate(&mut self) { unsafe { fdsp_bank_allocate(self.h, 64); } }                    // later process() calls do not allocate (audiounit.rs:92-95)
    fn set(&mut self, setting: Setting) {                                                     // audiounit.rs:62: address[0] = Index(voice)
        let mut s = setting;
        let voice = match s.direction() { Address::Index(i) => i as u32, _ => return };        // silently ignored like net.rs:1166
        s = s.peel();
        let (kind, vals): (c_int, Vec<f32>) = match s.parameter() {
            Parameter::Center(c) => (1, alloc::vec![*c]), Parameter::CenterQ(c, q) => (2, alloc::vec![*c, *q]), Parameter::CenterQGain(c, q, g) => (3, alloc::vec![*c, *q, *g]),
            Parameter::Value(v) => (4, alloc::vec![*v]), Parameter::Coefficient(c) => (5, alloc::vec![*c]),
            Parameter::Biquad(a1, a2, b0, b1, b2) => (6, alloc::vec![*a1, *a2, *b0, *b1, *b2]), Parameter::Delay(d) => (7, alloc::vec![*d]), Parameter::Time(t) => (8, alloc::vec![*t]),
            Parameter::Roughness(r) => (9, alloc::vec![*r]), Parameter::Variability(v) => (10, alloc::vec![*v]), Parameter::Pan(p) => (11, alloc::vec![*p]),
            Parameter::AttackRelease(a, r) => (12, alloc::vec![*a, *r]), _ => return,
        };
        let mut addr: Vec<i64> = Vec::new();                                                  // remaining address list: (1, index) | (2, node id) pairs
        loop {
            match s.direction() { Address::Left => { addr.push(1); addr.push(0); } Address::Right => { addr.push(1); addr.push(1); }
                                  Address::Index(i) => { addr.push(1); addr.push(i as i64); } Address::Node(id) => { addr.push(2); addr.push(id.value() as i64); } Address::Null => break }
            s = s.peel();
        }
        unsafe { fdsp_bank_set(self.h, voice, kind, vals.as_ptr(), vals.len() as c_int, 0, addr.as_ptr(), (addr.len() / 2) as c_int); }
    }
    fn process(&mut self, size: usize, input: &BufferRef, output: &mut BufferMut) {           // audiounit.rs:45
        // BufferRef / BufferMut are [channel][64] f32, 32-byte aligned (buffer.rs:12,156) == the ABI layout
        let ip = if self.inputs > 0 { input.channel_f32(0).as_ptr() } else { core::ptr::null() };
        let rc = unsafe { fdsp_bank_process(self.h, size as u32, ip, output.channel_f32_mut(0).as_mut_ptr()) };
        if rc != 0 { self.failed = true; for c in 0..self.outputs { output.channel_f32_mut(c)[..size].fill(0.0); } }   // process() has no error channel
    }
    fn tick(&mut self, input: &[f32], output: &mut [f32]) {
        let mut i = crate::buffer::BufferVec::new(self.inputs.max(1)); let mut o = crate::buffer::BufferVec::new(self.outputs);
        for (c, x) in input.iter().enumerate() { i.set_f32(c, 0, *x); }
        self.process(1, &i.buffer_ref(), &mut o.buffer_mut());
        for (c, y) in output.iter_mut().enumerate() { *y = o.at_f32(c, 0); }
    }
    fn get_id(&self) -> u64 { 1000 }
    fn ping(&mut self, _probe: bool, hash: AttoHash) -> AttoHash { hash.hash(self.get_id()) }
    fn route(&mut self, input: &SignalFrame, _frequency: f64) -> SignalFrame { Routing::Arbitrary(0.0).route(input, self.outputs()) }
    fn footprint(&self) -> usize { core::mem::size_of::<Self>() }
}
impl Clone for GpuBank {                                                                      // dyn_clone (audiounit.rs:373): deep copy incl. device state
    fn clone(&self) -> Self {
        let mut b: *mut FdspBank = core::ptr::null_mut();
        let rc = unsafe { fdsp_bank_clone(self.h, &mut b) };
        GpuBank { h: b, inputs: self.inputs, outputs: self.outputs, failed: self.failed || rc != 0 }
    }
}
impl Drop for GpuBank { fn drop(&mut self) { if !self.h.is_null() { unsafe { fdsp_bank_destroy(self.h) } } } }

/// The ranks whose banks are mixed down together (one process per GPU): voices shard, the ONE exchange step is the sum of the per-GPU
/// mixes, below the C ABI (NCCL gather over NVLink + rank-order fold). `id` comes from rank 0 (`GpuGroup::unique_id`) and reaches the
/// other ranks however the host likes (a file, a socket, MPI).
pub struct GpuGroup { h: *mut FdspGroup, pub rank: i32, pub nranks: i32 }
unsafe impl Send for GpuGroup {}
impl GpuGroup {
    pub fn unique_id() -> Result<[u8; 128], String> { let mut id = [0u8; 128]; check(unsafe { fdsp_group_unique_id(id.as_mut_ptr() as *mut c_void, 128) })?; Ok(id) }
    pub fn new(nranks: i32, rank: i32, id: &[u8; 128], device: i32) -> Result<Self, String> {
        let mut g: *mut FdspGroup = core::ptr::null_mut();
        check(unsafe { fdsp_group_create(nranks, rank, id.as_ptr() as *const c_void, device, &mut g) })?;
        Ok(GpuGroup { h: g, rank, nranks })
    }
    /// Every rank renders its shard; rank `root` receives the finished mix in `out` ([outputs][samples]).
    pub fn render_reduced(&self, bank: &mut GpuBank, samples: usize, input: Option<&[f32]>, out: Option<&mut [f32]>, root: i32) -> Result<(), String> {
        let op = out.map_or(core::ptr::null_mut(), |o| o.as_mut_ptr());
        check(unsafe { fdsp_bank_render_reduced(bank.h, self.h, samples as u64, input.map_or(core::ptr::null(), |x| x.as_ptr()), op, root) })
    }
}
impl Drop for GpuGroup { fn drop(&mut self) { if !self.h.is_null() { unsafe { fdsp_group_destroy(self.h) } } } }

/// VarFn with its closure text (gpu_var_fn!): the reference's node runs on the CPU side, the text lowers to the device over the Shared's cell.
pub struct GpuVarFn<X> { pub node: X, pub cell: alloc::sync::Arc<core::sync::atomic::AtomicU32>, pub text: &'static str, pub names: Vec<&'static str>, pub values: Vec<f32> }
impl<X: Clone> Clone for GpuVarFn<X> {
    fn clone(&self) -> Self { GpuVarFn { node: self.node.clone(), cell: self.cell.clone(), text: self.text, names: self.names.clone(), values: self.values.clone() } }
}
impl<X: AudioNode> AudioNode for GpuVarFn<X> {
    const ID: u64 = X::ID;
    type Inputs = X::Inputs;
    type Outputs = X::Outputs;
    fn reset(&mut self) { self.node.reset() }
    fn set_sample_rate(&mut self, sample_rate: f64) { self.node.set_sample_rate(sample_rate) }
    fn tick(&mut self, input: &Frame<f32, Self::Inputs>) -> Frame<f32, Self::Outputs> { self.node.tick(input) }
    fn process(&mut self, size: usize, input: &BufferRef, output: &mut BufferMut) { self.node.process(size, input, output) }
    fn set_hash(&mut self, hash: u64) { self.node.set_hash(hash) }
    fn route(&mut self, input: &SignalFrame, frequency: f64) -> SignalFrame { self.node.route(input, frequency) }
}
impl<X: AudioNode> Lower for GpuVarFn<X> {
    unsafe fn lower(&self) -> *mut FdspNode {
        let text: Vec<u8> = self.text.bytes().chain(core::iter::once(0)).collect();
        let names: Vec<Vec<u8>> = self.names.iter().map(|n| n.bytes().chain(core::iter::once(0)).collect()).collect();
        let ptrs: Vec<*const c_char> = names.iter().map(|n| n.as_ptr() as *const c_char).collect();
        let s = wrap_cell(&self.cell);
        let n = fdsp_var_fn(s, X::Outputs::I32, text.as_ptr() as *const c_char, self.values.len() as c_int, ptrs.as_ptr(), self.values.as_ptr());
        fdsp_shared_free(s);
        n
    }
}

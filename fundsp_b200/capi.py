"""ctypes binding of the C ABI (include/fundsp_b200.h) exported by fundsp_b200/libfundsp_b200.so.

The library is hand-written CUDA for sm_90a plus its host runtime; there is no CPU fallback: if the
shared object is missing or no CUDA device is usable the product path raises `FdspError`.
"""
from __future__ import annotations

import ctypes as C
import numpy as np
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.environ.get("FDSP_B200_LIB") or os.path.join(HERE, "libfundsp_b200.so")  # override: kernel build variants when tuning
HEADER = os.path.join(os.path.dirname(HERE), "include", "fundsp_b200.h")

OK, ERR_ARG, ERR_CUDA, ERR_UNSUPPORTED, ERR_ARITY, ERR_STATE = range(6)
OUT_VOICES, OUT_MIX = 1, 2


class FdspError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"fundsp_b200 error {code}: {msg}")
        self.code = code


_lib = None
P, F, D, I, U32, U64, I64 = C.c_void_p, C.c_float, C.c_double, C.c_int, C.c_uint32, C.c_uint64, C.c_int64
FP = C.POINTER(C.c_float)
ENVFN = C.CFUNCTYPE(None, C.c_double, C.POINTER(C.c_double), C.c_void_p)   # fdsp_envelope_fn
_KEEP = []   # ctypes callbacks handed to the library stay referenced for the life of the process


def envelope_callback(fn, outputs):
    """Wrap a Python closure `fn(t) -> float | tuple` as an fdsp_envelope_fn."""
    def cb(t, out, _user):
        v = fn(t)
        v = v if isinstance(v, (tuple, list)) else (v,)
        for i in range(outputs):
            out[i] = float(v[i])
    c = ENVFN(cb)
    _KEEP.append(c)
    return c

_SIG = {
    "fdsp_version": (C.c_char_p, []), "fdsp_last_error": (C.c_char_p, []), "fdsp_device_count": (I, []),
    "fdsp_constant": (P, [I, FP]), "fdsp_pass": (P, []), "fdsp_multipass": (P, [I]), "fdsp_sink": (P, [I]), "fdsp_split": (P, [I]),
    "fdsp_multisplit": (P, [I, I]), "fdsp_join": (P, [I]), "fdsp_multijoin": (P, [I, I]), "fdsp_reverse": (P, [I]), "fdsp_sine": (P, []),
    "fdsp_wavesynth": (P, [I, I]), "fdsp_noise": (P, []), "fdsp_fixed_svf": (P, [I, F, F, F]), "fdsp_svf": (P, [I, F, F, F]),
    "fdsp_sine_f64": (P, []), "fdsp_fixed_svf_f64": (P, [I, F, F, F]), "fdsp_svf_f64": (P, [I, F, F, F]),
    "fdsp_biquad_f64": (P, [F, F, F, F, F]), "fdsp_butterpass_f64": (P, [F, I]), "fdsp_resonator_f64": (P, [F, F, I]), "fdsp_onepole_f64": (P, [I, F, I]),
    "fdsp_biquad": (P, [F, F, F, F, F]), "fdsp_biquad_bank": (P, []), "fdsp_butterpass": (P, [F, I]), "fdsp_resonator": (P, [F, F, I]),
    "fdsp_moog": (P, [F, F, I]), "fdsp_fir": (P, [I, FP]), "fdsp_tick": (P, [I]), "fdsp_delay": (P, [D]), "fdsp_allnest": (P, [F, P, I]),
    "fdsp_phase_osc": (P, [I]), "fdsp_dsf": (P, [I, F, F]), "fdsp_reverb3": (P, [D, D, P]), "fdsp_var": (P, [F]), "fdsp_nl_biquad": (P, [I, I, I, F, F, I, F, F, F]), "fdsp_declick": (P, [F]), "fdsp_slot": (P, [P]), "fdsp_bank_slot_set": (I, [P, U32, I, D, P]), "fdsp_bank_crossfade_voice": (I, [P, U32, I, F, P]), "fdsp_oversample": (P, [P]), "fdsp_monitor": (P, []), "fdsp_envelope": (P, [D, I, I, ENVFN, P, D]), "fdsp_event": (P, [P, D, D, I, D, D]), "fdsp_event_loop": (P, [P, D, D, I, D, D, D]), "fdsp_limiter": (P, [I, F, F]), "fdsp_meter": (P, [I, D]), "fdsp_playwave": (P, [C.POINTER(C.c_float), C.c_uint64, C.c_uint64, C.c_uint64, C.c_int64]), "fdsp_resample": (P, [P]), "fdsp_phase_synth": (P, [I]), "fdsp_pulse": (P, []), "fdsp_mixer": (P, [I, I, C.POINTER(C.c_float)]), "fdsp_rotate": (P, [F, F]), "fdsp_chaos": (P, [I]), "fdsp_morph": (P, [F, F]), "fdsp_rez": (P, [F, F, F, I]), "fdsp_follow": (P, [I, F, F]), "fdsp_shaper": (P, [I, F, F]), "fdsp_onepole": (P, [I, F, I]), "fdsp_convolve": (P, [FP, I]), "fdsp_feedback_unit": (P, [D, P]), "fdsp_mls": (P, [I]), "fdsp_impulse": (P, [I]), "fdsp_tap": (P, [I, I, F, F]), "fdsp_feedback2": (P, [P, P, I]),
    "fdsp_pan": (P, [F]), "fdsp_panner": (P, []), "fdsp_adsr_live": (P, [F, F, F, F]),
    "fdsp_map": (P, [I, I, C.c_char_p, I, C.POINTER(C.c_char_p), FP]), "fdsp_shape_fn": (P, [C.c_char_p, I, C.POINTER(C.c_char_p), FP]),
    "fdsp_shaper_adaptive": (P, [D, I, F, F]), "fdsp_nl_biquad_adaptive": (P, [I, I, D, I, F, F, I, F, F, F]),
    "fdsp_envelope_in": (P, [D, I, I, C.c_char_p, I, C.POINTER(C.c_char_p), FP]),
    "fdsp_pipe": (P, [P, P]), "fdsp_stack": (P, [P, P]), "fdsp_branch": (P, [P, P]), "fdsp_bus": (P, [P, P]), "fdsp_thru": (P, [P]),
    "fdsp_binop": (P, [I, P, P]), "fdsp_unop": (P, [I, F, P]), "fdsp_multi": (P, [I, I, I, C.POINTER(P)]), "fdsp_feedback": (P, [P, I]),
    "fdsp_net_new": (P, [I, I]), "fdsp_net_push": (I, [P, P]), "fdsp_net_connect": (I, [P, I, I, I, I]), "fdsp_net_connect_input": (I, [P, I, I, I]),
    "fdsp_net_connect_output": (I, [P, I, I, I]), "fdsp_net_pass_through": (I, [P, I, I]), "fdsp_net_size": (I, [P]),
    "fdsp_node_phase": (I, [P, F]), "fdsp_node_seed": (I, [P, U64]), "fdsp_node_set": (I, [P, I, FP, I, U64, C.POINTER(I64), I]),
    "fdsp_node_inputs": (I, [P]), "fdsp_node_outputs": (I, [P]), "fdsp_node_id": (U64, [P]), "fdsp_node_ping": (U64, [P, I, U64]),
    "fdsp_node_leaf_hashes": (I, [P, C.POINTER(U64), I]), "fdsp_node_signature": (I, [P, C.c_char_p, I]), "fdsp_node_delay_floats": (C.c_int64, [P]), "fdsp_node_set_sample_rate": (I, [P, D]),
    "fdsp_node_lowering": (I, [P, C.POINTER(U32), I, C.POINTER(U32), I, C.POINTER(U32), I, C.POINTER(I), C.POINTER(I), C.POINTER(I)]), "fdsp_node_clone": (P, [P]), "fdsp_node_free": (None, [P]),
    "fdsp_wavetable_count": (I, [I]), "fdsp_wavetable_info": (I, [I, I, FP, C.POINTER(I)]), "fdsp_wavetable_data": (FP, [I, I]),
    "fdsp_bank_create": (I, [C.POINTER(P), U32, I, U32, C.POINTER(P)]), "fdsp_bank_create_from_net": (I, [P, I, U32, C.POINTER(P)]), "fdsp_bank_destroy": (None, [P]), "fdsp_bank_voice_of_vertex": (I, [P, I]), "fdsp_bank_clone": (I, [P, C.POINTER(P)]),
    "fdsp_bank_voices": (U32, [P]), "fdsp_bank_inputs": (I, [P]), "fdsp_bank_voice_outputs": (I, [P]), "fdsp_bank_outputs": (I, [P]),
    "fdsp_bank_set_sample_rate": (I, [P, D]), "fdsp_bank_reset": (I, [P]), "fdsp_bank_add_voice": (I, [P, P, C.POINTER(U32)]), "fdsp_jit_precompile": (I, [C.c_char_p, I, I]), "fdsp_bank_class_stages": (I, [P, I]),
    "fdsp_group_unique_id": (I, [P, U64]), "fdsp_group_create": (I, [I, I, P, I, C.POINTER(P)]), "fdsp_group_destroy": (None, [P]), "fdsp_group_rank": (I, [P]), "fdsp_group_size": (I, [P]),
    "fdsp_bank_render_reduced": (I, [P, P, U64, FP, FP, I]), "fdsp_bank_reduce_device": (I, [P, P, U64, P, U64, I]), "fdsp_jit_cache_stats": (None, [C.POINTER(I), C.POINTER(I)]), "fdsp_wave_save": (I, [C.c_char_p, FP, U32, U64, U64, D, I]), "fdsp_wave_encode": (C.c_int64, [C.POINTER(C.c_uint8), U64, FP, U32, U64, U64, D, I]), "fdsp_wave_load": (I, [C.c_char_p, FP, U64, C.POINTER(U32), C.POINTER(U64), C.POINTER(D)]), "fdsp_bank_edit_event": (I, [P, U32, D, D]), "fdsp_bank_push_event": (I, [P, P, C.POINTER(U32)]), "fdsp_bank_replace_voice": (I, [P, U32, P]), "fdsp_bank_remove_voice": (I, [P, U32]), "fdsp_bank_time": (D, [P]), "fdsp_bank_set": (I, [P, U32, I, FP, I, U64, C.POINTER(I64), I]), "fdsp_bank_allocate": (I, [P, U64]),
    "fdsp_bank_process": (I, [P, U32, FP, FP]), "fdsp_bank_render": (I, [P, U64, FP, FP, FP]),
    "fdsp_bank_render_device": (I, [P, U64, P, U64, P, U64, P, U64]), "fdsp_bank_sync": (I, [P]), "fdsp_bank_stream": (P, [P]),
    "fdsp_bank_num_classes": (I, [P]), "fdsp_bank_class_info": (I, [P, I, C.c_char_p, I, C.POINTER(U32), C.POINTER(U32), C.POINTER(U32), C.POINTER(U64)]),
    "fdsp_bank_launch_count": (U64, [P]), "fdsp_bank_last_kernel_ms": (F, [P]), "fdsp_bank_last_dominant_ms": (F, [P]),
}


def header_symbols():
    """Every function name declared in include/fundsp_b200.h."""
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(fdsp_[a-z0-9_]+)\s*\(", text)))


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            raise FdspError(ERR_STATE, f"{SO} is missing: build it with `make -C fundsp_b200/csrc` (or __graft_entry__.build()); there is no CPU fallback")
        L = C.CDLL(SO)
        for name, (res, args) in _SIG.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(code):
    if code != OK:
        raise FdspError(code, lib().fdsp_last_error().decode())


def _node(h, what):
    if not h:
        raise FdspError(ERR_ARITY, lib().fdsp_last_error().decode() or what)
    return h


def _farr(v):
    if hasattr(v, "__array__"):   # a wave channel: no per-element conversion (data_as keeps the array alive)
        return np.ascontiguousarray(np.asarray(v, dtype=np.float32)).ctypes.data_as(C.POINTER(C.c_float))
    return (C.c_float * len(v))(*v)


def _caps(caps):
    """Captured values as the C ABI takes them: count, names, f32 values."""
    names = [k.encode() for k, _ in caps]
    return len(caps), (C.c_char_p * max(1, len(caps)))(*names), (C.c_float * max(1, len(caps)))(*[v for _, v in caps])


def _closure_node(h):
    """A closure node handle, or the refusal: ArityError for an arity mismatch (the reference's compile-time error), else FdspError."""
    if not h:
        msg = lib().fdsp_last_error().decode()
        if ": arity mismatch" in msg:
            from .graph import ArityError
            raise ArityError(msg)
        raise FdspError(ERR_ARG, msg)
    return h


class GpuBackend:
    """Lowers `An` expressions to fdsp_node handles (one `b_<op>` per primitive in fundsp_b200/graph.py)."""

    def __init__(self):
        self.L = lib()

    def b_constant(self, v): return _node(self.L.fdsp_constant(len(v), _farr(v)), "constant")
    def b_pass(self): return _node(self.L.fdsp_pass(), "pass")
    def b_multipass(self, n): return _node(self.L.fdsp_multipass(n), "multipass")
    def b_sink(self, n): return _node(self.L.fdsp_sink(n), "sink")
    def b_split(self, n): return _node(self.L.fdsp_split(n), "split")
    def b_multisplit(self, m, n): return _node(self.L.fdsp_multisplit(m, n), "multisplit")
    def b_join(self, n): return _node(self.L.fdsp_join(n), "join")
    def b_multijoin(self, m, n): return _node(self.L.fdsp_multijoin(m, n), "multijoin")
    def b_reverse(self, n): return _node(self.L.fdsp_reverse(n), "reverse")
    def b_sine(self): return _node(self.L.fdsp_sine(), "sine")
    def b_wavesynth(self, kind, nout): return _node(self.L.fdsp_wavesynth(kind, nout), "wavesynth")
    def b_noise(self): return _node(self.L.fdsp_noise(), "noise")
    def b_fixed_svf(self, mode, f, q, g): return _node(self.L.fdsp_fixed_svf(mode, f, q, g), "fixed_svf")
    def b_svf(self, mode, f, q, g): return _node(self.L.fdsp_svf(mode, f, q, g), "svf")
    def b_sine_f64(self): return _node(self.L.fdsp_sine_f64(), "sine_f64")
    def b_fixed_svf_f64(self, mode, f, q, g): return _node(self.L.fdsp_fixed_svf_f64(mode, f, q, g), "fixed_svf_f64")
    def b_svf_f64(self, mode, f, q, g): return _node(self.L.fdsp_svf_f64(mode, f, q, g), "svf_f64")
    def b_biquad_f64(self, a1, a2, b0, b1, b2): return _node(self.L.fdsp_biquad_f64(a1, a2, b0, b1, b2), "biquad_f64")
    def b_butterpass_f64(self, f, nin): return _node(self.L.fdsp_butterpass_f64(f, nin), "butterpass_f64")
    def b_resonator_f64(self, f, q, nin): return _node(self.L.fdsp_resonator_f64(f, q, nin), "resonator_f64")
    def b_onepole_f64(self, kind, param, nin): return _node(self.L.fdsp_onepole_f64(kind, param, nin), "onepole_f64")
    def b_biquad(self, a1, a2, b0, b1, b2): return _node(self.L.fdsp_biquad(a1, a2, b0, b1, b2), "biquad")
    def b_biquad_bank(self): return _node(self.L.fdsp_biquad_bank(), "biquad_bank")
    def b_butterpass(self, f, nin): return _node(self.L.fdsp_butterpass(f, nin), "butterpass")
    def b_resonator(self, f, q, nin): return _node(self.L.fdsp_resonator(f, q, nin), "resonator")
    def b_moog(self, f, q, nin): return _node(self.L.fdsp_moog(f, q, nin), "moog")
    def b_fir(self, w): return _node(self.L.fdsp_fir(len(w), _farr(w)), "fir")
    def b_tick(self, n): return _node(self.L.fdsp_tick(n), "tick")
    def b_delay(self, t): return _node(self.L.fdsp_delay(t), "delay")
    def b_allnest(self, c, nin, x): return _node(self.L.fdsp_allnest(c, x, nin), "allnest")
    def b_phase_osc(self, kind): return _node(self.L.fdsp_phase_osc(kind), "phase_osc")
    def b_reverb3(self, time, diffusion, filt): return _node(self.L.fdsp_reverb3(time, diffusion, filt), "reverb3")
    def b_feedback_unit(self, delay, x): return _node(self.L.fdsp_feedback_unit(delay, x), "feedback_unit")
    def b_convolve(self, response): return _node(self.L.fdsp_convolve(_farr(response), len(response)), "convolve")
    def b_onepole(self, kind, param, nin): return _node(self.L.fdsp_onepole(kind, param, nin), "onepole")
    def b_shaper(self, kind, p0, p1): return _node(self.L.fdsp_shaper(kind, p0, p1), "shaper")
    def b_follow(self, asym, a, r): return _node(self.L.fdsp_follow(asym, a, r), "follow")
    def b_morph(self, cutoff, q): return _node(self.L.fdsp_morph(cutoff, q), "morph")
    def b_rez(self, bp, cutoff, q, nin): return _node(self.L.fdsp_rez(bp, cutoff, q, nin), "rez")
    def b_chaos(self, kind): return _node(self.L.fdsp_chaos(kind), "chaos")
    def b_declick(self, d): return _node(self.L.fdsp_declick(d), "declick")
    def b_slot(self, x): return _node(self.L.fdsp_slot(x), "slot")
    def b_oversample(self, x): return _node(self.L.fdsp_oversample(x), "oversample")
    def b_monitor(self): return _node(self.L.fdsp_monitor(), "monitor")
    def b_envelope(self, interval, nout, t64, fn, horizon): return _node(self.L.fdsp_envelope(interval, nout, t64, envelope_callback(fn, nout), None, horizon), "envelope")
    def b_event(self, start, end, ease, fi, fo, x): return _node(self.L.fdsp_event(x, start, end, ease, fi, fo), "event")
    def b_event_loop(self, start, end, ease, fi, fo, loop, x): return _node(self.L.fdsp_event_loop(x, start, end, ease, fi, fo, loop), "event_loop")
    def b_limiter(self, n, a, r): return _node(self.L.fdsp_limiter(n, a, r), "limiter")
    def b_meter(self, kind, timescale): return _node(self.L.fdsp_meter(kind, timescale), "meter")
    def b_playwave(self, samples, start, end, loop): return _node(self.L.fdsp_playwave(_farr(samples), len(samples), start, end, loop), "playwave")
    def b_resample(self, x): return _node(self.L.fdsp_resample(x), "resample")
    def b_phase_synth(self, kind): return _node(self.L.fdsp_phase_synth(kind), "phase_synth")
    def b_pulse(self): return _node(self.L.fdsp_pulse(), "pulse")
    def b_mixer(self, m, n, w): return _node(self.L.fdsp_mixer(m, n, _farr(w)), "mixer")
    def b_rotate(self, angle, gain): return _node(self.L.fdsp_rotate(angle, gain), "rotate")
    def b_netnode(self, net): return net.lower(self)
    def b_nl_biquad(self, fb, mode, shape, p0, p1, nin, ce, q, g): return _node(self.L.fdsp_nl_biquad(fb, mode, shape, p0, p1, nin, ce, q, g), "nl_biquad")
    def b_shaper_adaptive(self, timescale, kind, p0, p1): return _node(self.L.fdsp_shaper_adaptive(timescale, kind, p0, p1), "shaper_adaptive")
    def b_nl_biquad_adaptive(self, fb, mode, timescale, kind, p0, p1, nin, ce, q, g):
        return _node(self.L.fdsp_nl_biquad_adaptive(fb, mode, timescale, kind, p0, p1, nin, ce, q, g), "nl_biquad_adaptive")
    def b_var(self, value): return _node(self.L.fdsp_var(value), "var")
    def b_dsf(self, n, spacing, rough): return _node(self.L.fdsp_dsf(n, spacing, rough), "dsf")
    def b_mls(self, bits): return _node(self.L.fdsp_mls(bits), "mls")
    def b_impulse(self, n): return _node(self.L.fdsp_impulse(n), "impulse")
    def b_tap(self, n, lin, mn, mx): return _node(self.L.fdsp_tap(n, lin, mn, mx), "tap")
    def b_feedback2(self, had, x, y): return _node(self.L.fdsp_feedback2(x, y, had), "feedback2")
    def b_pan(self, p): return _node(self.L.fdsp_pan(p), "pan")
    def b_panner(self): return _node(self.L.fdsp_panner(), "panner")
    def b_adsr_live(self, a, d, s, r): return _node(self.L.fdsp_adsr_live(a, d, s, r), "adsr_live")
    def b_map(self, text, nin, nout, caps): return _closure_node(self.L.fdsp_map(nin, nout, text.encode(), *_caps(caps)))
    def b_shape_fn(self, text, caps): return _closure_node(self.L.fdsp_shape_fn(text.encode(), *_caps(caps)))
    def b_envelope_in(self, interval, text, nin, nout, caps): return _closure_node(self.L.fdsp_envelope_in(interval, nin, nout, text.encode(), *_caps(caps)))
    def b_pipe(self, x, y): return _node(self.L.fdsp_pipe(x, y), "pipe")
    def b_stack(self, x, y): return _node(self.L.fdsp_stack(x, y), "stack")
    def b_branch(self, x, y): return _node(self.L.fdsp_branch(x, y), "branch")
    def b_bus(self, x, y): return _node(self.L.fdsp_bus(x, y), "bus")
    def b_thru(self, x): return _node(self.L.fdsp_thru(x), "thru")
    def b_binop(self, op, x, y): return _node(self.L.fdsp_binop(op, x, y), "binop")
    def b_unop(self, kind, s, x): return _node(self.L.fdsp_unop(kind, s, x), "unop")
    def b_multi(self, kind, op, n, *nodes): return _node(self.L.fdsp_multi(kind, op, n, (C.c_void_p * n)(*nodes)), "multi")
    def b_feedback(self, had, x): return _node(self.L.fdsp_feedback(x, had), "feedback")

    def b_phase(self, p, x):
        check(self.L.fdsp_node_phase(x, p))
        return x

    # Net container (fundsp_b200/net.py)
    def net_new(self, i, o): return _node(self.L.fdsp_net_new(i, o), "net_new")

    def net_push(self, net, unit):
        idx = self.L.fdsp_net_push(net, unit)
        if idx < 0:
            raise FdspError(ERR_ARG, "net_push failed")
        return idx

    def net_connect(self, net, s, sp, t, tp): check(self.L.fdsp_net_connect(net, s, sp, t, tp))
    def net_connect_input(self, net, gi, t, tp): check(self.L.fdsp_net_connect_input(net, gi, t, tp))
    def net_connect_output(self, net, s, sp, go): check(self.L.fdsp_net_connect_output(net, s, sp, go))
    def net_pass_through(self, net, gi, go): check(self.L.fdsp_net_pass_through(net, gi, go))

    def b_seed(self, s, x):
        check(self.L.fdsp_node_seed(x, s))
        return x

    def b_set(self, kind, values, seed, address, x):
        addr = [v for pair in address for v in pair]
        check(self.L.fdsp_node_set(x, kind, _farr(values), len(values), seed, (C.c_int64 * max(1, len(addr)))(*addr), len(address)))
        return x


class NodeHandle:
    """Owns an fdsp_node built from an `An` expression (host-side description; no GPU needed)."""

    def __init__(self, expr):
        self.L = lib()
        self.h = expr.lower(GpuBackend())

    def __del__(self):
        try:
            if self.h:
                self.L.fdsp_node_free(self.h)
        except Exception:
            pass

    def take(self):
        h, self.h = self.h, None
        return h

    def inputs(self): return self.L.fdsp_node_inputs(self.h)
    def outputs(self): return self.L.fdsp_node_outputs(self.h)
    def ping(self, probe, h): return self.L.fdsp_node_ping(self.h, 1 if probe else 0, h)

    def leaf_hashes(self):
        buf = (C.c_uint64 * 4096)()
        n = self.L.fdsp_node_leaf_hashes(self.h, buf, 4096)
        return [int(buf[i]) for i in range(n)]

    def lowering(self):
        """(P, S, U) words of the device program, in load order (numpy uint32 arrays)."""
        import numpy as np
        n = [C.c_int(0), C.c_int(0), C.c_int(0)]
        check(self.L.fdsp_node_lowering(self.h, None, 0, None, 0, None, 0, C.byref(n[0]), C.byref(n[1]), C.byref(n[2])))
        arrs = [np.zeros(max(1, x.value), np.uint32) for x in n]
        ptr = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))
        check(self.L.fdsp_node_lowering(self.h, ptr(arrs[0]), len(arrs[0]), ptr(arrs[1]), len(arrs[1]), ptr(arrs[2]), len(arrs[2]), C.byref(n[0]), C.byref(n[1]), C.byref(n[2])))
        return tuple(a[: x.value] for a, x in zip(arrs, n))

    def set_sample_rate(self, sr):
        check(self.L.fdsp_node_set_sample_rate(self.h, float(sr)))

    def delay_floats(self):
        return int(self.L.fdsp_node_delay_floats(self.h))

    def signature(self):
        buf = C.create_string_buffer(1 << 16)
        self.L.fdsp_node_signature(self.h, buf, len(buf))
        return buf.value.decode()


# ---- Wave files (src/write.rs): planar [channels, n] f32 arrays <-> the reference's WAV bytes
def save_wav(path, wave, sample_rate, bits=16):
    """Wave::save_wav16 / save_wav32."""
    w = np.ascontiguousarray(np.atleast_2d(np.asarray(wave, np.float32)))
    check(lib().fdsp_wave_save(str(path).encode(), w.ctypes.data_as(FP), w.shape[0], w.shape[1], w.shape[1], float(sample_rate), int(bits)))


def encode_wav(wave, sample_rate, bits=16):
    """Wave::write_wav16 / write_wav32 into memory."""
    w = np.ascontiguousarray(np.atleast_2d(np.asarray(wave, np.float32)))
    L = lib()
    n = L.fdsp_wave_encode(None, 0, w.ctypes.data_as(FP), w.shape[0], w.shape[1], w.shape[1], float(sample_rate), int(bits))
    if n < 0:
        check(ERR_ARG)
    buf = (C.c_uint8 * n)()
    L.fdsp_wave_encode(buf, n, w.ctypes.data_as(FP), w.shape[0], w.shape[1], w.shape[1], float(sample_rate), int(bits))
    return bytes(buf)


def load_wav(path):
    """Returns (wave[channels, n], sample_rate)."""
    L = lib()
    ch, n, sr = U32(0), U64(0), D(0.0)
    check(L.fdsp_wave_load(str(path).encode(), None, 0, C.byref(ch), C.byref(n), C.byref(sr)))
    w = np.zeros((ch.value, n.value), np.float32)
    check(L.fdsp_wave_load(str(path).encode(), w.ctypes.data_as(FP), w.size, C.byref(ch), C.byref(n), C.byref(sr)))
    return w, sr.value


def jit_precompile(signature, mode, table_variant=0):
    """Compile one unit of a graph class into the on-disk JIT cache (no GPU needed)."""
    check(lib().fdsp_jit_precompile(signature.encode(), int(mode), int(table_variant)))


def jit_cache_stats():
    h, r = I(0), I(0)
    lib().fdsp_jit_cache_stats(C.byref(h), C.byref(r))
    return {"hits": h.value, "nvrtc_runs": r.value}

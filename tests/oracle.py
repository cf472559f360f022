"""ctypes binding of the CPU oracle (oracle/_build/libfundsp_oracle.so) — TEST INFRASTRUCTURE.

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs import this module.
`OracleBackend` lowers a `fundsp_b200.graph.An` expression onto the oracle's node classes.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile
import weakref

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ODIR = os.path.join(ROOT, "oracle")
SO = os.path.join(ODIR, "_build", "libfundsp_oracle.so")


def build_oracle():
    """The oracle library, built by oracle/Makefile when it is missing or older than any oracle source. A tree that cannot be
    written and holds no up-to-date library gets one built in a per-user temporary directory instead."""
    so = SO
    if not os.access(ODIR, os.W_OK) and subprocess.call(["make", "-q", "-C", ODIR], stdout=subprocess.DEVNULL) != 0:
        so = os.path.join(tempfile.gettempdir(), f"fdsp_oracle_{os.getuid()}", "libfundsp_oracle.so")
    subprocess.check_call(["make", "-C", ODIR, "OUT=" + so], stdout=subprocess.DEVNULL)
    return so


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(os.environ.get("FDSP_ORACLE_SO") or build_oracle())   # FDSP_ORACLE_SO: bench.py's -march=native build for the TIMED CPU arm only
        P, F, D, I, U64, I64 = C.c_void_p, C.c_float, C.c_double, C.c_int, C.c_uint64, C.c_int64
        FP, S = C.POINTER(C.c_float), C.c_char_p
        sig = {
            "fo_about": (C.c_char_p, []),
            "fo_rnd1": (D, [U64]), "fo_hash1": (U64, [U64]), "fo_attohash": (U64, [U64, U64]), "fo_hash32x": (C.c_uint32, [C.c_uint32]),
            "fo_wide_sinf": (F, [F]), "fo_wide_floorf": (F, [F]), "fo_lerpf": (F, [F, F, F]), "fo_lerpd": (D, [D, D, D]),
            "fo_delerpd": (D, [D, D, D]), "fo_xerpf": (F, [F, F, F]), "fo_xerpd": (D, [D, D, D]), "fo_db_amp": (D, [D]), "fo_smooth9f": (F, [F]),
            "fo_set_denormal_emulation": (None, [I]), "fo_restore_denormals": (None, []),
            "fo_wavetable_count": (I, [I]), "fo_wavetable_pitch": (F, [I, I]), "fo_wavetable_len": (I, [I, I]), "fo_wavetable_data": (FP, [I, I]),
            "fo_wavetable_install": (I, [I, I, FP, C.POINTER(I), FP]), "fo_wavetable_restore": (None, [I]),
            "fo_constant": (P, [I, FP]), "fo_pass": (P, []), "fo_multipass": (P, [I]), "fo_sink": (P, [I]), "fo_split": (P, [I]),
            "fo_multisplit": (P, [I, I]), "fo_join": (P, [I]), "fo_multijoin": (P, [I, I]), "fo_reverse": (P, [I]), "fo_sine": (P, []),
            "fo_wavesynth": (P, [I, I]), "fo_noise": (P, []), "fo_fixed_svf": (P, [I, F, F, F]), "fo_svf": (P, [I, F, F, F]),
            "fo_biquad": (P, [F, F, F, F, F]), "fo_biquad_bank": (P, []), "fo_butterpass": (P, [F, I]), "fo_resonator": (P, [F, F, I]),
            "fo_moog": (P, [F, F, I]), "fo_fir": (P, [I, FP]), "fo_tick_node": (P, [I]), "fo_delay": (P, [D]), "fo_allnest": (P, [F, P, I]),
            "fo_phase_osc": (P, [I]), "fo_dsf": (P, [I, F, F]), "fo_reverb3": (P, [D, D, P]), "fo_var": (P, [F]), "fo_nl_biquad": (P, [I, I, I, F, F, I, F, F, F]), "fo_declick": (P, [F]), "fo_slot": (P, [P]), "fo_slot_set": (None, [P, I, D, P]), "fo_oversample": (P, [P]), "fo_monitor": (P, []), "fo_envelope": (P, [D, I, I, C.CFUNCTYPE(None, C.c_double, C.POINTER(C.c_double), C.c_void_p), P]), "fo_sequencer": (P, [I, I, I, D]), "fo_sequencer_push": (C.c_uint64, [P, D, D, I, D, D, P]), "fo_sequencer_push_relative": (C.c_uint64, [P, D, D, I, D, D, P]), "fo_sequencer_edit": (None, [P, C.c_uint64, D, D]), "fo_sequencer_edit_relative": (None, [P, C.c_uint64, D, D]), "fo_sequencer_time": (D, [P]), "fo_limiter": (P, [I, F, F]), "fo_meter": (P, [I, D]), "fo_playwave": (P, [C.POINTER(C.c_float), C.c_uint64, C.c_uint64, C.c_uint64, C.c_int64]), "fo_resample": (P, [P]), "fo_phase_synth": (P, [I]), "fo_pulse": (P, []), "fo_mixer": (P, [I, I, C.POINTER(C.c_float)]), "fo_rotate": (P, [F, F]), "fo_chaos": (P, [I]), "fo_morph": (P, [F, F]), "fo_rez": (P, [F, F, F, I]), "fo_follow": (P, [I, F, F]), "fo_shaper": (P, [I, F, F]), "fo_onepole": (P, [I, F, I]), "fo_convolve": (P, [FP, I]), "fo_feedback_unit": (P, [D, P]), "fo_libm_eval": (None, [I, FP, FP, FP, C.c_int64]), "fo_mls": (P, [I]), "fo_impulse": (P, [I]), "fo_tap": (P, [I, I, F, F]), "fo_feedback2": (P, [P, P, I]),
            "fo_pan": (P, [F]), "fo_panner": (P, []), "fo_adsr_live": (P, [F, F, F, F]), "fo_biquad_coefs": (None, [I, F, F, F, F, FP]),
            "fo_pipe": (P, [P, P]), "fo_stack": (P, [P, P]), "fo_branch": (P, [P, P]), "fo_bus": (P, [P, P]), "fo_thru": (P, [P]),
            "fo_binop": (P, [I, P, P]), "fo_unop": (P, [I, F, P]), "fo_multi": (P, [I, I, I, C.POINTER(P)]), "fo_feedback": (P, [P, I]),
            "fo_sine_hz": (P, [F]), "fo_wave_hz": (P, [I, F]), "fo_fir3": (P, [F]), "fo_moog_q": (P, [F]), "fo_reverb_stereo": (P, [D, D, D]),
            "fo_phase": (None, [P, F]), "fo_seed": (None, [P, U64]), "fo_set": (None, [P, I, FP, I, U64, C.POINTER(I64), I]),
            "fo_inputs": (I, [P]), "fo_outputs": (I, [P]), "fo_id": (U64, [P]), "fo_reset": (None, [P]), "fo_set_sample_rate": (None, [P, D]),
            "fo_tick": (None, [P, FP, FP]), "fo_process": (None, [P, I, FP, FP]), "fo_ping": (U64, [P, I, U64]), "fo_set_hash": (None, [P, U64]),
            "fo_clone": (P, [P]), "fo_leaf_hashes": (I, [P, C.POINTER(U64), I]), "fo_free": (None, [P]),
            "fo_render_length": (I64, [D, D]), "fo_render": (None, [P, D, D, FP]), "fo_filter": (None, [P, D, FP, I64, I64, FP]),
            "fo_process_many": (None, [P, I64, FP, FP]),
            "fo_net_new": (P, [I, I]), "fo_net_wrap": (P, [P]), "fo_net_push": (I, [P, P]), "fo_net_chain": (I, [P, P]),
            "fo_net_connect": (None, [P, I, I, I, I]), "fo_net_connect_input": (None, [P, I, I, I]), "fo_net_connect_output": (None, [P, I, I, I]),
            "fo_net_pipe_input": (None, [P, I]), "fo_net_pipe_output": (None, [P, I]), "fo_net_pipe_all": (None, [P, I, I]),
            "fo_net_pass_through": (None, [P, I, I]), "fo_net_size": (I, [P]), "fo_net_has_cycle": (I, [P]), "fo_net_order": (I, [P, C.POINTER(I)]),
            "fo_net_combine": (P, [I, P, P]), "fo_net_crossfade": (None, [P, I, I, F, P]),
            "fo_bank_render": (None, [C.POINTER(P), I64, D, I64, FP, FP, FP, I]),
            # fo_shapes.cpp: the Atan and Adaptive waveshapes
            "fo_atanf": (F, [F]), "fo_wide_atanf": (F, [F]), "fo_shaper_x": (P, [I, F, F]), "fo_shaper_adaptive": (P, [D, I, F, F]),
            "fo_nl_biquad_x": (P, [I, I, I, F, F, I, F, F, F]), "fo_nl_biquad_adaptive": (P, [I, I, D, I, F, F, I, F, F, F]),
            # fo_closure.cpp: closures of the signal
            "fo_map": (P, [I, I, S, I, C.POINTER(S), FP]), "fo_shape_fn": (P, [S, I, C.POINTER(S), FP]),
            "fo_envelope_in": (P, [D, I, I, S, I, C.POINTER(S), FP]),
            # fo_prelude64.cpp: the prelude64 nodes and the f64 libm
            "fo64_sin": (D, [D]), "fo64_cos": (D, [D]), "fo64_tan": (D, [D]), "fo64_exp": (D, [D]),
            "fo64_rem_pio2_medium": (I, [D, C.POINTER(D)]), "fo64_rem_pio2_large": (I, [D, C.POINTER(D)]),
            "fo64_eval": (None, [I, C.POINTER(D), C.POINTER(D), I64]),
            "fo_sine_f64": (P, []), "fo_fixed_svf_f64": (P, [I, F, F, F]), "fo_svf_f64": (P, [I, F, F, F]),
            "fo_biquad_f64": (P, [F, F, F, F, F]), "fo_butterpass_f64": (P, [F, I]), "fo_resonator_f64": (P, [F, F, I]),
            "fo_onepole_f64": (P, [I, F, I]), "fo_sine_f64_phase_after": (D, [U64, D, F, I]),
            # fo_shared.cpp: Shared cells and the nodes that read and write them
            "fo_shared_new": (P, [F]), "fo_shared_free": (None, [P]), "fo_shared_set": (None, [P, F]), "fo_shared_get": (F, [P]),
            "fo_var_shared": (P, [P]), "fo_monitor_shared": (P, [P, I, D]), "fo_timer": (P, [P]),
            "fo_var_fn": (P, [P, I, S, I, C.POINTER(S), FP]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float)) if a is not None else None


def _farr(v):
    if hasattr(v, "__array__"):   # a wave channel: no per-element conversion (data_as keeps the array alive)
        return np.ascontiguousarray(np.asarray(v, dtype=np.float32)).ctypes.data_as(C.POINTER(C.c_float))
    return (C.c_float * len(v))(*v)


def _caps(caps):
    """A closure's captures as the oracle takes them: count, names, values."""
    names = [k.encode() for k, _ in caps]
    return len(caps), (C.c_char_p * max(1, len(caps)))(*names), (C.c_float * max(1, len(caps)))(*[v for _, v in caps])


def _node(h):
    if not h:
        raise ValueError("the oracle has no such node, or its closure interpreter could not parse the closure")
    return h


class OracleBackend:
    """Lowers `An` expressions to oracle nodes (one `b_<op>` per primitive in fundsp_b200/graph.py)."""

    def __init__(self):
        self.L = lib()

    def b_constant(self, v): return self.L.fo_constant(len(v), _farr(v))
    def b_pass(self): return self.L.fo_pass()
    def b_multipass(self, n): return self.L.fo_multipass(n)
    def b_sink(self, n): return self.L.fo_sink(n)
    def b_split(self, n): return self.L.fo_split(n)
    def b_multisplit(self, m, n): return self.L.fo_multisplit(m, n)
    def b_join(self, n): return self.L.fo_join(n)
    def b_multijoin(self, m, n): return self.L.fo_multijoin(m, n)
    def b_reverse(self, n): return self.L.fo_reverse(n)
    def b_sine(self): return self.L.fo_sine()
    def b_wavesynth(self, kind, nout): return self.L.fo_wavesynth(kind, nout)
    def b_noise(self): return self.L.fo_noise()
    def b_fixed_svf(self, mode, f, q, g): return self.L.fo_fixed_svf(mode, f, q, g)
    def b_svf(self, mode, f, q, g): return self.L.fo_svf(mode, f, q, g)
    def b_biquad(self, a1, a2, b0, b1, b2): return self.L.fo_biquad(a1, a2, b0, b1, b2)
    def b_biquad_bank(self): return self.L.fo_biquad_bank()
    def b_butterpass(self, f, nin): return self.L.fo_butterpass(f, nin)
    def b_resonator(self, f, q, nin): return self.L.fo_resonator(f, q, nin)
    def b_moog(self, f, q, nin): return self.L.fo_moog(f, q, nin)
    def b_fir(self, w): return self.L.fo_fir(len(w), _farr(w))
    def b_tick(self, n): return self.L.fo_tick_node(n)
    def b_delay(self, t): return self.L.fo_delay(t)
    def b_allnest(self, c, nin, x): return self.L.fo_allnest(c, x, nin)
    def b_phase_osc(self, kind): return self.L.fo_phase_osc(kind)
    def b_reverb3(self, time, diffusion, filt): return self.L.fo_reverb3(time, diffusion, filt)
    def b_feedback_unit(self, delay, x): return self.L.fo_feedback_unit(delay, x)
    def b_convolve(self, response): return self.L.fo_convolve(_farr(response), len(response))
    def b_onepole(self, kind, param, nin): return self.L.fo_onepole(kind, param, nin)
    def b_shaper(self, kind, p0, p1): return _node(self.L.fo_shaper_x(kind, p0, p1)) if kind == 6 else self.L.fo_shaper(kind, p0, p1)   # 6: Atan
    def b_shaper_adaptive(self, timescale, kind, p0, p1): return _node(self.L.fo_shaper_adaptive(timescale, kind, p0, p1))
    def b_follow(self, asym, a, r): return self.L.fo_follow(asym, a, r)
    def b_morph(self, cutoff, q): return self.L.fo_morph(cutoff, q)
    def b_rez(self, bp, cutoff, q, nin): return self.L.fo_rez(bp, cutoff, q, nin)
    def b_chaos(self, kind): return self.L.fo_chaos(kind)
    def b_declick(self, d): return self.L.fo_declick(d)
    def b_slot(self, x): return self.L.fo_slot(x)
    def b_oversample(self, x): return self.L.fo_oversample(x)
    def b_monitor(self): return self.L.fo_monitor()
    def b_envelope(self, interval, nout, t64, fn, horizon):   # the oracle calls the closure live, like the reference (no horizon)
        from fundsp_b200.capi import envelope_callback
        return self.L.fo_envelope(interval, nout, t64, envelope_callback(fn, nout), None)
    def b_event(self, start, end, ease, fi, fo, x):   # the checker for one event is a one-event Sequencer (ReplayMode::All)
        h = self.L.fo_sequencer(0, self.L.fo_outputs(x), 0, 0.0)
        self.L.fo_sequencer_push(h, start, end, ease, fi, fo, x)
        return h
    def b_event_loop(self, start, end, ease, fi, fo, loop, x):   # ... of a ReplayMode::Loop(loop) sequencer (mode 2)
        h = self.L.fo_sequencer(0, self.L.fo_outputs(x), 2, loop)
        self.L.fo_sequencer_push(h, start, end, ease, fi, fo, x)
        return h
    def b_limiter(self, n, a, r): return self.L.fo_limiter(n, a, r)
    def b_meter(self, kind, timescale): return self.L.fo_meter(kind, timescale)
    def b_playwave(self, samples, start, end, loop): return self.L.fo_playwave(_farr(samples), len(samples), start, end, loop)
    def b_resample(self, x): return self.L.fo_resample(x)
    def b_phase_synth(self, kind): return self.L.fo_phase_synth(kind)
    def b_pulse(self): return self.L.fo_pulse()
    def b_mixer(self, m, n, w): return self.L.fo_mixer(m, n, _farr(w))
    def b_rotate(self, angle, gain): return self.L.fo_rotate(angle, gain)
    def b_netnode(self, net): return net.lower(self)
    def b_seqnode(self, seq): return seq.lower(self)
    def sequencer_new(self, i, o, mode, loop): return self.L.fo_sequencer(i, o, mode, loop)
    def sequencer_push(self, h, s, e, ease, fi, fo, unit, rel): return (self.L.fo_sequencer_push_relative if rel else self.L.fo_sequencer_push)(h, s, e, ease, fi, fo, unit)
    def sequencer_edit(self, h, eid, end, fo, rel): (self.L.fo_sequencer_edit_relative if rel else self.L.fo_sequencer_edit)(h, eid, end, fo)
    def b_nl_biquad(self, fb, mode, shape, p0, p1, nin, ce, q, g):
        return (_node(self.L.fo_nl_biquad_x(fb, mode, shape, p0, p1, nin, ce, q, g)) if shape == 6 else
                self.L.fo_nl_biquad(fb, mode, shape, p0, p1, nin, ce, q, g))
    def b_nl_biquad_adaptive(self, fb, mode, timescale, kind, p0, p1, nin, ce, q, g):
        return _node(self.L.fo_nl_biquad_adaptive(fb, mode, timescale, kind, p0, p1, nin, ce, q, g))
    def b_var(self, value): return self.L.fo_var(value)
    def b_dsf(self, n, spacing, rough): return self.L.fo_dsf(n, spacing, rough)
    def b_mls(self, bits): return self.L.fo_mls(bits)
    def b_impulse(self, n): return self.L.fo_impulse(n)
    def b_tap(self, n, lin, mn, mx): return self.L.fo_tap(n, lin, mn, mx)
    def b_feedback2(self, had, x, y): return self.L.fo_feedback2(x, y, had)
    def b_pan(self, p): return self.L.fo_pan(p)
    def b_panner(self): return self.L.fo_panner()
    def b_adsr_live(self, a, d, s, r): return self.L.fo_adsr_live(a, d, s, r)
    def b_pipe(self, x, y): return self.L.fo_pipe(x, y)
    def b_stack(self, x, y): return self.L.fo_stack(x, y)
    def b_branch(self, x, y): return self.L.fo_branch(x, y)
    def b_bus(self, x, y): return self.L.fo_bus(x, y)
    def b_thru(self, x): return self.L.fo_thru(x)
    def b_binop(self, op, x, y): return self.L.fo_binop(op, x, y)
    def b_unop(self, kind, s, x): return self.L.fo_unop(kind, s, x)
    def b_multi(self, kind, op, n, *nodes): return self.L.fo_multi(kind, op, n, (C.c_void_p * n)(*nodes))
    def b_feedback(self, had, x): return self.L.fo_feedback(x, had)
    def b_phase(self, p, x): self.L.fo_phase(x, p); return x
    def b_seed(self, s, x): self.L.fo_seed(x, s); return x
    # closures of the signal (fo_closure.h)
    def b_map(self, text, nin, nout, caps): return _node(self.L.fo_map(nin, nout, text.encode(), *_caps(caps)))
    def b_shape_fn(self, text, caps): return _node(self.L.fo_shape_fn(text.encode(), *_caps(caps)))
    def b_envelope_in(self, interval, text, nin, nout, caps): return _node(self.L.fo_envelope_in(interval, nin, nout, text.encode(), *_caps(caps)))
    # prelude64 (fo_prelude64.h)
    def b_sine_f64(self): return _node(self.L.fo_sine_f64())
    def b_fixed_svf_f64(self, mode, f, q, g): return _node(self.L.fo_fixed_svf_f64(mode, f, q, g))
    def b_svf_f64(self, mode, f, q, g): return _node(self.L.fo_svf_f64(mode, f, q, g))
    def b_biquad_f64(self, a1, a2, b0, b1, b2): return _node(self.L.fo_biquad_f64(a1, a2, b0, b1, b2))
    def b_butterpass_f64(self, f, nin): return _node(self.L.fo_butterpass_f64(f, nin))
    def b_resonator_f64(self, f, q, nin): return _node(self.L.fo_resonator_f64(f, q, nin))
    def b_onepole_f64(self, kind, p, nin): return _node(self.L.fo_onepole_f64(kind, p, nin))
    # Shared controls (fo_shared.h), each on the oracle cell that mirrors the product's Shared
    def b_var_shared(self, s): return _node(self.L.fo_var_shared(mirror(s).h))
    def b_monitor_shared(self, s, kind, timescale): return _node(self.L.fo_monitor_shared(mirror(s).h, kind, timescale))
    def b_timer(self, s): return _node(self.L.fo_timer(mirror(s).h))
    def b_var_fn(self, s, text, nout, caps): return _node(self.L.fo_var_fn(mirror(s).h, nout, text.encode(), *_caps(caps)))
    # Net container (fundsp_b200/net.py)
    def net_new(self, i, o): return self.L.fo_net_new(i, o)
    def net_push(self, net, unit): return self.L.fo_net_push(net, unit)
    def net_connect(self, net, s, sp, t, tp): self.L.fo_net_connect(net, s, sp, t, tp)
    def net_connect_input(self, net, gi, t, tp): self.L.fo_net_connect_input(net, gi, t, tp)
    def net_connect_output(self, net, s, sp, go): self.L.fo_net_connect_output(net, s, sp, go)
    def net_pass_through(self, net, gi, go): self.L.fo_net_pass_through(net, gi, go)

    def b_set(self, kind, values, seed, address, x):
        addr = [v for pair in address for v in pair]
        self.L.fo_set(x, kind, _farr(values), len(values), seed, (C.c_int64 * max(1, len(addr)))(*addr), len(address))
        return x


class OracleUnit:
    """An oracle graph as an `AudioUnit`: render / filter / process / tick."""

    def __init__(self, expr_or_handle):
        self.L = lib()
        self.h = expr_or_handle.lower(OracleBackend()) if hasattr(expr_or_handle, "lower") else expr_or_handle

    def __del__(self):
        try:
            if self.h:
                self.L.fo_free(self.h)
        except Exception:
            pass

    def take(self):
        h, self.h = self.h, None
        return h

    def inputs(self): return self.L.fo_inputs(self.h)
    def outputs(self): return self.L.fo_outputs(self.h)
    def reset(self): self.L.fo_reset(self.h)
    def set_sample_rate(self, sr): self.L.fo_set_sample_rate(self.h, sr)
    def ping(self, probe, h): return self.L.fo_ping(self.h, 1 if probe else 0, h)

    def leaf_hashes(self):
        buf = (C.c_uint64 * 4096)()
        n = self.L.fo_leaf_hashes(self.h, buf, 4096)
        return [int(buf[i]) for i in range(n)]

    def render(self, sr, duration):
        n = self.L.fo_render_length(sr, duration)
        out = np.zeros((self.outputs(), n), np.float32)
        self.L.fo_render(self.h, sr, duration, _fp(out))
        return out

    def filter(self, sr, inp, total=None):
        inp = np.ascontiguousarray(inp, np.float32).reshape(self.inputs(), -1)
        total = inp.shape[1] if total is None else total
        out = np.zeros((self.outputs(), total), np.float32)
        self.L.fo_filter(self.h, sr, _fp(inp), inp.shape[1], total, _fp(out))
        return out

    def process_many(self, n, inp=None):
        if inp is None:
            inp = np.zeros((max(1, self.inputs()), n), np.float32)
        inp = np.ascontiguousarray(inp, np.float32)
        out = np.zeros((self.outputs(), n), np.float32)
        self.L.fo_process_many(self.h, n, _fp(inp), _fp(out))
        return out

    def process(self, size, inp=None):
        ib = np.zeros((max(1, self.inputs()), 64), np.float32)
        if inp is not None:
            ib[: self.inputs(), :size] = np.asarray(inp, np.float32).reshape(self.inputs(), -1)[:, :size]
        ob = np.zeros((max(1, self.outputs()), 64), np.float32)
        self.L.fo_process(self.h, size, _fp(ib), _fp(ob))
        return ob[: self.outputs(), :size].copy()

    def tick(self, frame=()):
        fi = np.zeros(max(1, self.inputs()), np.float32)
        fi[: len(frame)] = frame
        fo = np.zeros(max(1, self.outputs()), np.float32)
        self.L.fo_tick(self.h, _fp(fi), _fp(fo))
        return fo[: self.outputs()].copy()


class OracleShared:
    """An oracle cell (std::shared_ptr<std::atomic<uint32_t>>)."""

    def __init__(self, value=0.0):
        self.h = lib().fo_shared_new(value)

    def set(self, v): lib().fo_shared_set(self.h, v)
    def value(self): return float(lib().fo_shared_get(self.h))

    def __del__(self):
        try:
            lib().fo_shared_free(self.h)
        except Exception:  # noqa: BLE001
            pass


_MIRRORS = weakref.WeakKeyDictionary()


def mirror(s):
    """The oracle cell that stands for the product Shared `s`: each product `Shared` gets one of its own, created with the product
    cell's value on first use, so a test drives both sides with `set_both` and compares `s.value()` with `mirror(s).value()`."""
    m = _MIRRORS.get(s)
    if m is None:
        m = _MIRRORS[s] = OracleShared(s.value())
    return m


def set_both(s, v):
    s.set(v)
    mirror(s).set(v)


def oracle_bank_render(exprs, sr, n, inp=None, per_voice=True, mix=False, threads=1):
    """CPU 'bank' = a Vec of units + index-order sum (SURVEY.md §3.6). Returns (out[V,c,n] | None, mix[c,n] | None)."""
    L = lib()
    be = OracleBackend()
    hs = [e.lower(be) for e in exprs]
    V = len(hs)
    no, ni = L.fo_outputs(hs[0]), L.fo_inputs(hs[0])
    arr = (C.c_void_p * V)(*hs)
    out = np.zeros((V, no, n), np.float32) if per_voice else None
    mx = np.zeros((no, n), np.float32) if mix else None
    ib = np.zeros((max(1, ni), n), np.float32) if inp is None else np.ascontiguousarray(inp, np.float32).reshape(max(1, ni), n)
    import time
    t0 = time.perf_counter()
    L.fo_bank_render(arr, V, sr, n, _fp(ib), _fp(out), _fp(mx), threads)
    oracle_bank_render.last_seconds = time.perf_counter() - t0  # render only (graph construction excluded)
    for h in hs:
        L.fo_free(h)
    return out, mx

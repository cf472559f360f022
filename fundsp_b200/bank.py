"""GpuBank: V voice instances of FunDSP graphs evaluated in lockstep on one H100.

To the host it is one `AudioUnit` (reference src/audiounit.rs:21-95) with `inputs()` shared bus inputs
and either 2-ish mixed outputs (`mix=True`) or `V * channels` per-voice outputs: `process` is
`AudioUnit::process`, `render`/`filter` are `Wave::render` / `Wave::filter` (src/wave.rs:441-466,518-565).
Its CPU equivalent in the reference is "a Vec of V units + a sum" (SURVEY.md §3.6).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi
from .capi import OUT_MIX, OUT_VOICES, FdspError, GpuBackend, check


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float)) if a is not None else None


class GpuBank:
    def __init__(self, voices, device=0, per_voice=True, mix=False, sample_rate=None):
        """`voices`: sequence of `An` expressions (one per voice; they may fall into several structural classes)."""
        self.L = capi.lib()
        be = GpuBackend()
        hs = [v.lower(be) for v in voices]
        mode = (OUT_VOICES if per_voice else 0) | (OUT_MIX if mix else 0)
        out = C.c_void_p()
        arr = (C.c_void_p * len(hs))(*hs)
        check(self.L.fdsp_bank_create(arr, len(hs), device, mode, C.byref(out)))
        self.h = out
        self.mode = mode
        self.device = device
        if sample_rate is not None:
            self.set_sample_rate(sample_rate)

    @classmethod
    def from_net(cls, net, device=0, per_voice=False, mix=True, sample_rate=None):
        """Bank from a voice-separable `Net` (voice vertices + `Net::bus` adder trees): the mix-down follows the Net's own
        association order bit for bit and voices get the phase hashes of `Net::ping`."""
        self = object.__new__(cls)
        self.L = capi.lib()
        h = net.lower(GpuBackend())
        mode = (OUT_VOICES if per_voice else 0) | (OUT_MIX if mix else 0)
        out = C.c_void_p()
        check(self.L.fdsp_bank_create_from_net(h, device, mode, C.byref(out)))
        self.h, self.mode, self.device = out, mode, device
        if sample_rate is not None:
            self.set_sample_rate(sample_rate)
        return self

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.L.fdsp_bank_destroy(self.h)
                self.h = None
        except Exception:
            pass

    # ---- AudioUnit surface
    def voices(self): return self.L.fdsp_bank_voices(self.h)
    def inputs(self): return self.L.fdsp_bank_inputs(self.h)
    def voice_outputs(self): return self.L.fdsp_bank_voice_outputs(self.h)
    def outputs(self): return self.L.fdsp_bank_outputs(self.h)
    def set_sample_rate(self, sr): check(self.L.fdsp_bank_set_sample_rate(self.h, float(sr)))
    def voice_of_vertex(self, vertex): return self.L.fdsp_bank_voice_of_vertex(self.h, int(vertex))

    def reset(self): check(self.L.fdsp_bank_reset(self.h))

    def set(self, voice, kind, values=(), seed=0, address=()):
        """AudioUnit::set on one voice: `kind` is a setting.rs Parameter index (capi.P_*), `address` = [(1, index) | (2, node_id), ...]."""
        import ctypes as C
        addr = [x for pair in address for x in pair]
        vals = (C.c_float * max(1, len(values)))(*values)
        check(self.L.fdsp_bank_set(self.h, voice, kind, vals, len(values), seed, (C.c_int64 * max(1, len(addr)))(*addr), len(address)))

    # ---- sequencer banks (voices built with fundsp_b200.sequencer.event): the mix output is Sequencer::process
    @classmethod
    def from_sequencer(cls, seq, device=0, per_voice=False, mix=True, sample_rate=None):
        """One voice per pushed event (`Sequencer.voices()`), in push order."""
        return cls(seq.voices(), device=device, per_voice=per_voice, mix=mix, sample_rate=sample_rate)

    def time(self):
        """Sequencer::time: seconds rendered since the last reset (the f64 clock every event voice keeps on the device)."""
        return float(self.L.fdsp_bank_time(self.h))

    def edit_event(self, voice, end_time, fade_out_time):
        """Sequencer::edit on a live bank."""
        check(self.L.fdsp_bank_edit_event(self.h, int(voice), float(end_time), float(fade_out_time)))

    def push_event(self, ev):
        """Sequencer::push on a running bank: `ev` (an `event(...)` expression) takes the slot of a finished event of the same
        graph class, or — when there is none — the bank grows by one voice (`add_voice`); returns the voice index."""
        v = C.c_uint32(0)
        check(self.L.fdsp_bank_push_event(self.h, ev.lower(GpuBackend()), C.byref(v)))
        return int(v.value)

    def slot_set(self, voice, fade_ease, fade_time, unit):
        """Slot::set on a voice built with `slot(unit)`: crossfade to `unit` (same graph class) over fade_time seconds."""
        check(self.L.fdsp_bank_slot_set(self.h, int(voice), int(fade_ease), float(fade_time), unit.lower(GpuBackend())))

    def add_voice(self, unit):
        """Grow the bank by one voice (running state of the others preserved; O(bank state)); returns its index."""
        v = C.c_uint32(0)
        check(self.L.fdsp_bank_add_voice(self.h, unit.lower(GpuBackend()), C.byref(v)))
        return int(v.value)

    def replace_voice(self, voice, unit):
        """`Net::replace`: any unit of the bank's arity in the voice's place (fresh state); another graph class regroups the classes around it."""
        check(self.L.fdsp_bank_replace_voice(self.h, int(voice), unit.lower(GpuBackend())))

    def crossfade_voice(self, voice, fade_ease, fade_time, unit):
        """`Net::crossfade`: the voice fades to `unit` (any graph class of the bank's arity) over fade_time seconds, Fade.Power (0) or Fade.Smooth (1)."""
        check(self.L.fdsp_bank_crossfade_voice(self.h, int(voice), int(fade_ease), float(fade_time), unit.lower(GpuBackend())))

    def remove_voice(self, voice):
        """`Net::remove`: the voice carries silence from now on (its place in the mix order stays)."""
        check(self.L.fdsp_bank_remove_voice(self.h, int(voice)))

    def allocate(self, max_samples=64): check(self.L.fdsp_bank_allocate(self.h, int(max_samples)))

    def clone(self):
        out = C.c_void_p()
        check(self.L.fdsp_bank_clone(self.h, C.byref(out)))
        b = object.__new__(GpuBank)
        b.L, b.h, b.mode, b.device = self.L, out, self.mode, self.device
        return b

    def process(self, size, inp=None):
        """AudioUnit::process: returns [outputs, size] (mix if the bank mixes, else V*channels rows)."""
        ni = self.inputs()
        ib = np.zeros((max(1, ni), 64), np.float32)
        if inp is not None and ni:
            ib[:ni, :size] = np.asarray(inp, np.float32).reshape(ni, -1)[:, :size]
        ob = np.zeros((self.outputs(), 64), np.float32)
        check(self.L.fdsp_bank_process(self.h, size, _fp(ib), _fp(ob)))
        return ob[:, :size].copy()

    def render(self, sample_rate, duration, inp=None):
        """Wave::render (no inputs) / Wave::filter (inputs): returns (voices[V, c, n] | None, mix[c, n] | None)."""
        self.set_sample_rate(sample_rate)
        n = int(round(duration * sample_rate))
        return self.render_samples(n, inp)

    def render_samples(self, n, inp=None):
        ni, c, V = self.inputs(), self.voice_outputs(), self.voices()
        ib = None
        if ni:
            ib = np.zeros((ni, n), np.float32)
            if inp is not None:
                x = np.asarray(inp, np.float32).reshape(ni, -1)
                ib[:, : min(n, x.shape[1])] = x[:, :n]
        ov = np.zeros((V * c, n), np.float32) if self.mode & OUT_VOICES else None
        om = np.zeros((c, n), np.float32) if self.mode & OUT_MIX else None
        check(self.L.fdsp_bank_render(self.h, n, _fp(ib), _fp(ov), _fp(om)))
        return (ov.reshape(V, c, n) if ov is not None else None), om

    def render_device(self, n, in_ptr=0, in_stride=0, out_ptr=0, out_stride=0, mix_ptr=0, mix_stride=0, sync=True):
        """Device-resident render (raw device pointers, strides in floats); asynchronous unless sync."""
        check(self.L.fdsp_bank_render_device(self.h, n, in_ptr, in_stride, out_ptr, out_stride, mix_ptr, mix_stride))
        if sync:
            self.sync()

    def sync(self): check(self.L.fdsp_bank_sync(self.h))
    def stream(self): return self.L.fdsp_bank_stream(self.h)
    def launch_count(self): return int(self.L.fdsp_bank_launch_count(self.h))
    def last_kernel_ms(self): return float(self.L.fdsp_bank_last_kernel_ms(self.h))
    def last_dominant_ms(self): return float(self.L.fdsp_bank_last_dominant_ms(self.h))

    def classes(self):
        out = []
        for i in range(self.L.fdsp_bank_num_classes(self.h)):
            sig = C.create_string_buffer(1 << 16)
            v, s, p, d = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint64()
            check(self.L.fdsp_bank_class_info(self.h, i, sig, len(sig), C.byref(v), C.byref(s), C.byref(p), C.byref(d)))
            out.append(dict(signature=sig.value.decode(), voices=v.value, state_words=s.value, param_words=p.value, delay_floats=d.value,
                            stages=self.L.fdsp_bank_class_stages(self.h, i)))
        return out


__all__ = ["GpuBank", "FdspError"]

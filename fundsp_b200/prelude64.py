"""Opcode vocabulary of the reference's `prelude64` (src/prelude64.rs, F = f64): the "audio hacking" environment, where filters and
oscillators keep their internal state in f64.

`from fundsp_b200.prelude64 import *` gives every name of `fundsp_b200.prelude`; the ones whose prelude64 type carries `f64` are
replaced here. Arguments stay f32 (the reference converts them with `F::from_f32`), and so do node inputs and outputs.

Lowered with f64 state: `sine`/`sine_hz` (`Sine<f64>`), the nine SVF modes in every form (`FixedSvf<f64, M>` for `x_hz`,
`Svf<f64, M>` for `x()` and `x_q`), `biquad`, `butterpass(_hz)`, `resonator(_hz)`, `lowpole(_hz)`, `highpole(_hz)`,
`allpole(_delay)`, `dcblock(_hz)`, `pinkpass`, `pink` and `brown`. `envelope`/`lfo` are the f64-time envelopes (`time64=True`).

Every other name whose prelude64 type is f64 raises `NotImplementedError` naming that type: an f32 node in its place would compute
something else, so it is never substituted.
"""
from __future__ import annotations

from . import prelude as _p32
from .graph import An, f32
from .prelude import *  # noqa: F401,F403
from .prelude import (ALLPASS, BANDPASS, BELL, HIGHPASS, HIGHSHELF, LOWPASS, LOWSHELF, NOTCH, PEAK, dc, multipass, white)


# ---- src/prelude64.rs:338-351
def sine():
    return An("sine_f64", (), (), 1, 1)


def sine_hz(f):
    return dc(f) >> sine()


# ---- src/prelude64.rs:1917-2140 Simper SVF family with F = f64
def _svf(mode):
    return An("svf_f64", (mode, 440.0, 1.0, 1.0), (), 4 if mode >= BELL else 3, 1)


def _svf_hz(mode, f, q, gain=1.0):
    return An("fixed_svf_f64", (mode, f32(f), f32(q), f32(gain)), (), 1, 1)


def _svf_q(mode, q, gain=None):
    n = An("svf_f64", (mode, 440.0, f32(q), 1.0 if gain is None else f32(gain)), (), 3 if gain is None else 4, 1)
    return (multipass(2) | (dc(q) if gain is None else dc((q, gain)))) >> n


def lowpass(): return _svf(LOWPASS)
def lowpass_hz(f, q): return _svf_hz(LOWPASS, f, q)
def lowpass_q(q): return _svf_q(LOWPASS, q)
def highpass(): return _svf(HIGHPASS)
def highpass_hz(f, q): return _svf_hz(HIGHPASS, f, q)
def highpass_q(q): return _svf_q(HIGHPASS, q)
def bandpass(): return _svf(BANDPASS)
def bandpass_hz(f, q): return _svf_hz(BANDPASS, f, q)
def bandpass_q(q): return _svf_q(BANDPASS, q)
def notch(): return _svf(NOTCH)
def notch_hz(f, q): return _svf_hz(NOTCH, f, q)
def notch_q(q): return _svf_q(NOTCH, q)
def peak(): return _svf(PEAK)
def peak_hz(f, q): return _svf_hz(PEAK, f, q)
def peak_q(q): return _svf_q(PEAK, q)
def allpass(): return _svf(ALLPASS)
def allpass_hz(f, q): return _svf_hz(ALLPASS, f, q)
def allpass_q(q): return _svf_q(ALLPASS, q)
def bell(): return _svf(BELL)
def bell_hz(f, q, gain): return _svf_hz(BELL, f, q, gain)
def bell_q(q, gain): return _svf_q(BELL, q, gain)
def lowshelf(): return _svf(LOWSHELF)
def lowshelf_hz(f, q, gain): return _svf_hz(LOWSHELF, f, q, gain)
def lowshelf_q(q, gain): return _svf_q(LOWSHELF, q, gain)
def highshelf(): return _svf(HIGHSHELF)
def highshelf_hz(f, q, gain): return _svf_hz(HIGHSHELF, f, q, gain)
def highshelf_q(q, gain): return _svf_q(HIGHSHELF, q, gain)


# ---- src/prelude64.rs:442-541: biquads and one-poles with F = f64
def biquad(a1, a2, b0, b1, b2):
    return An("biquad_f64", (f32(a1), f32(a2), f32(b0), f32(b1), f32(b2)), (), 1, 1)


def butterpass():
    return An("butterpass_f64", (440.0, 2), (), 2, 1)


def butterpass_hz(f):
    return An("butterpass_f64", (f32(f), 1), (), 1, 1)


def resonator():
    return An("resonator_f64", (440.0, 1.0, 3), (), 3, 1)


def resonator_hz(center, q):
    return An("resonator_f64", (f32(center), f32(q), 1), (), 1, 1)


def lowpole():
    return An("onepole_f64", (0, 440.0, 2), (), 2, 1)


def lowpole_hz(cutoff):
    return An("onepole_f64", (0, f32(cutoff), 1), (), 1, 1)


def highpole():
    return An("onepole_f64", (1, 440.0, 2), (), 2, 1)


def highpole_hz(cutoff):
    return An("onepole_f64", (1, f32(cutoff), 1), (), 1, 1)


def allpole():
    return An("onepole_f64", (2, 1.0, 2), (), 2, 1)


def allpole_delay(delay_in_samples):
    return An("onepole_f64", (2, f32(delay_in_samples), 1), (), 1, 1)


# ---- src/prelude64.rs:1147-1160, 1293-1310
def dcblock_hz(cutoff):
    return An("onepole_f64", (3, f32(cutoff), 1), (), 1, 1)


def dcblock():
    return dcblock_hz(10.0)


def pinkpass():
    return An("onepole_f64", (4, 0.0, 1), (), 1, 1)


def pink():
    return white() >> pinkpass()


def brown():
    return white() >> lowpole_hz(10.0) * dc(13.7)


# ---- src/prelude64.rs:581-612: Envelope<f64, E, R>
def envelope(f, outputs=None, horizon=10.0, interval=0.002):
    return _p32.envelope(f, outputs, horizon, True, interval)


def lfo(f, outputs=None, horizon=10.0):
    return _p32.envelope(f, outputs, horizon, True)


# ---- names whose prelude64 type is f64 and has no f64 lowering here
_F64_ONLY = {
    "biquad_bank": "BiquadBank<f64x4>",
    "moog": "Moog<f64, U3>", "moog_q": "Moog<f64, U3>", "moog_hz": "Moog<f64, U1>",
    "lowrez": "Rez<f64, U3>", "lowrez_hz": "Rez<f64, U1>", "lowrez_q": "Rez<f64, U3>", "bandrez": "Rez<f64, U3>",
    "bandrez_hz": "Rez<f64, U1>", "bandrez_q": "Rez<f64, U3>", "morph": "Morph<f64>", "morph_hz": "Morph<f64>",
    "follow": "Follow<f64>", "afollow": "AFollow<f64>", "declick": "Declick<f64>", "declick_s": "Declick<f64>",
    "ramp": "Ramp<f64>", "ramp_hz": "Ramp<f64>", "poly_saw": "PolySaw<f64>", "poly_saw_hz": "PolySaw<f64>",
    "poly_square": "PolySquare<f64>", "poly_square_hz": "PolySquare<f64>", "poly_pulse": "PolyPulse<f64>", "poly_pulse_hz": "PolyPulse<f64>",
    "envelope_in": "EnvelopeIn<f64, E, I, R>", "lfo_in": "EnvelopeIn<f64, E, I, R>", "envelope2": "EnvelopeIn<f64, E, U1, R>",
    "lfo2": "EnvelopeIn<f64, E, U1, R>", "envelope3": "EnvelopeIn<f64, E, U2, R>", "lfo3": "EnvelopeIn<f64, E, U2, R>",
    **{f"{d}{m}{hz}": f"{'DirtyBiquad' if d == 'd' else 'FbBiquad'}<f64, {m.capitalize()}Biquad<f64>, S>"
       for d in "df" for m in ("bell", "highpass", "lowpass", "resonator") for hz in ("", "_hz")},
}


def _refuse(name, ty):
    def f(*_args, **_kw):
        raise NotImplementedError(f"{name}: prelude64 builds {ty}, which has no f64 lowering in fundsp_b200 yet "
                                  f"(use fundsp_b200.prelude for the f32 form)")
    f.__name__ = name
    return f


for _name, _ty in _F64_ONLY.items():
    globals()[_name] = _refuse(_name, _ty)
del _name, _ty

"""Text envelopes without a GPU: the `|t|` closure kind (accepted and refused texts), canonical class signatures and one class for voices
that differ in captures, the oracle's Envelope running a text through its closure interpreter pinned bit for bit against the same
Envelope running numpy float32 callbacks, NVRTC compilation of every class of tests/test_gpu_envelope_text.py for sm_90a, the device node
on the host emulation against the oracle, the GPU file on the CPU mock device, and a lowering without sampled values."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from fundsp_b200 import capi, prelude64
from fundsp_b200.capi import FdspError
from fundsp_b200.graph import ArityError
from fundsp_b200.prelude import *  # noqa: F401,F403
from oracle import OracleUnit, lib as olib
from test_mock_bank_cpu import ROOT, mock_env  # noqa: F401  (the mock device build, shared with that file)

import test_gpu_envelope_text as G

F32 = np.float32
P_INTERVAL = 15


def sig(g):
    return capi.NodeHandle(g).signature()


# ---- 1. the language: |t| only, the arity of the value, captures
ACCEPTED = [
    ("|t| t", 1),
    ("move |t: f32| -t * 0.5", 1),
    ("|time| { let a = time * 2.0; (a, a * a, sin(a)) }", 3),
    ("|t| if t < 1.0 { (t, 1.0) } else { (1.0, t) }", 2),
    ("|t| lerp(0.0, 1.0, clamp01(t)) + sqr_hz(2.0, t) + tri_hz(1.0, t) + sin_hz(3.0, t) + cos_hz(1.0, t)", 1),
    ("|t| (t, t, t, t, t, t, t, t)", 8),
]

REFUSED = [   # (text, outputs, exception, the message must contain)
    ("|t, x| t * x", 1, ArityError, "envelope: arity mismatch: envelope takes one time parameter |t|, the text has 2 parameters"),
    ("|| 1.0", 1, ArityError, "envelope takes one time parameter |t|, the text has 0 parameters"),
    ("|t| (t, t)", 1, ArityError, "arity mismatch: the closure returns 2 values, the node has 1 output"),
    ("|t| t", 2, ArityError, "arity mismatch: the closure returns 1 value, the node has 2 outputs"),
    ("|t| t", 9, ArityError, "arity mismatch: 0-8 inputs and 1-8 outputs"),
    ("|t| t[0]", 1, FdspError, "`[` at column 6: only a frame parameter can be indexed"),
    ("|t| t * k", 1, FdspError, "`k` is neither a parameter nor a captured value"),
    ("|t| log(t)", 1, FdspError, "`log` at column 5: its musl source is not restated"),
    ("|t| t.atan()", 1, FdspError, "`atan` at column 7: its musl source is not restated"),
    ("|t| t * 2", 1, FdspError, "`2` at column 9: integer literals are not supported"),
    ("|t| t as f32", 1, FdspError, "`as` at column 7: `as` casts are not supported"),
]


@pytest.mark.parametrize("text,nout", ACCEPTED)
def test_accepted_texts(text, nout):
    h = capi.NodeHandle(envelope(text, nout))
    assert h.inputs() == 0 and h.outputs() == nout and h.signature().startswith(f"EnvelopeFn<{nout},0,Ex::")
    assert capi.lib().fdsp_node_id(h.h) == 14


@pytest.mark.parametrize("text,nout,exc,msg", REFUSED)
def test_refused_texts(text, nout, exc, msg):
    with pytest.raises(exc) as e:
        envelope(text, nout)
    assert msg in str(e.value), str(e.value)
    if exc is FdspError:
        assert e.value.code == capi.ERR_ARG


def test_refusals_of_captures_and_of_other_forms():
    with pytest.raises(FdspError, match="envelope: capture `k` does not occur in the closure"):
        lfo("|t| t", k=1.0)
    with pytest.raises(FdspError, match="the interval must be positive"):
        envelope("|t| t", interval=0.0)
    with pytest.raises(TypeError, match="captured values are for a text closure"):
        envelope(lambda t: t, k=1.0)
    for f in (prelude64.envelope, prelude64.lfo, lambda text: envelope(text, time64=True)):
        with pytest.raises(NotImplementedError, match="f64"):
            f("|t| t")
    lib = capi.lib()
    assert not lib.fdsp_envelope_text(0.002, 1, b"|t| t * k", 0, None, None)
    assert b"`k` is neither a parameter" in lib.fdsp_last_error()


# ---- 2. canonical signatures, captures as per-voice words, one class
def test_signatures_are_canonical():
    a = lfo("|t| sin_hz(rate, t) * depth", rate=1.0, depth=0.5)
    b = lfo("move |time: f32|   sin_hz( rate,time ) * depth // vibrato", rate=7.0, depth=-2.0)
    assert sig(a) == sig(b) == "EnvelopeFn<1,2,Ex::Mul<Ex::SinHz<Ex::Cap<0>,Ex::T>,Ex::Cap<1>>>"
    assert sig(lfo("|t| t * 0.5")) == sig(envelope("|s| s * 5e-1")) != sig(lfo("|t| t * 0.25"))
    assert sig(lfo("|t| t * k", k=1.0)) != sig(lfo("|t| t * 1.0"))
    P, S, U = capi.NodeHandle(lfo("|t| t * b + a", a=2.0, b=3.0)).lowering()
    assert list(P.view(F32)) == [3.0, 2.0, F32(0.002)] and len(U) == 0      # captures in order of first occurrence, then the interval
    assert len(S) == 8 + 4 * 1


def test_one_class_for_sixteen_thousand_voices_on_the_mock_device(mock_env):
    code = ("from fundsp_b200.bank import GpuBank\nfrom fundsp_b200.prelude import lfo, sine\n"
            "b = GpuBank([lfo('|t| 100.0 + 10.0 * sin_hz(r, t)', r=0.5 + i / 16384.0) >> sine() for i in range(16384)], per_voice=False, mix=True)\n"
            "print('classes', b.L.fdsp_bank_num_classes(b.h), b.voices())\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=mock_env, cwd=ROOT, timeout=900)
    assert r.returncode == 0 and "classes 1 16384" in r.stdout, (r.stdout[-500:], r.stderr[-1500:])


def test_no_table_words_whatever_the_render_length():
    """The text form's parameter words are its captures and interval, for any render length; the callback form stores one word per
    output and sample point up to its horizon."""
    text = lambda: envelope("|t| (t * a, t - a, 1.0)", 3, a=0.5)
    P, _, _ = capi.NodeHandle(text()).lowering()
    assert len(P) == 2
    cb = lambda hz: envelope(lambda t: (t * 0.5, t - 0.5, 1.0), 3, horizon=hz)
    p10, p60 = (len(capi.NodeHandle(cb(hz)).lowering()[0]) for hz in (10.0, 60.0))
    assert p10 > 3 * 4000 and p60 > 5 * p10


# ---- 3. the oracle's Envelope running the text (its interpreter as the live closure) against the same Envelope running numpy float32
EXACT = [   # (text, outputs, captures, numpy float32 form of the same operations)
    ("|t| t * a + 0.25", 1, dict(a=1.5), lambda t, a: (t * a + F32(0.25),)),
    ("|t| { let u = t * 3.0; (u - floor(u), min(t, a), max(t * t, 0.5)) }", 3, dict(a=0.3),
     lambda t, a: (t * F32(3.0) - np.floor(t * F32(3.0)), np.fmin(t, a), np.fmax(t * t, F32(0.5)))),
    ("|t| if t < a { t / a } else { (1.0 - t) * 2.0 }", 1, dict(a=0.2), lambda t, a: (t / a if t < a else (F32(1.0) - t) * F32(2.0),)),
    ("|t| (lerp(-1.0, 1.0, clamp01(t * a)), sqrt(t), abs(t - 0.5))", 3, dict(a=4.0),
     lambda t, a: (F32(-1.0) * (F32(1.0) - np.fmin(np.fmax(t * a, F32(0.0)), F32(1.0))) + F32(1.0) * np.fmin(np.fmax(t * a, F32(0.0)), F32(1.0)),
                   np.sqrt(t), np.abs(t - F32(0.5)))),
]


def _numpy_callback(f, a):
    def cb(t):
        with np.errstate(all="ignore"):
            v = f(F32(t), F32(a))
        return tuple(float(F32(x)) for x in v) if len(v) > 1 else float(F32(v[0]))
    return cb


@pytest.mark.parametrize("k", range(len(EXACT)))
@pytest.mark.parametrize("sr", [44100.0, 48000.0])
def test_oracle_text_envelope_equals_callback_envelope(k, sr):
    text, nout, caps, f = EXACT[k]
    olib().fo_set_denormal_emulation(0)
    us = [OracleUnit(G.oracle_of(envelope(text, nout, **caps))), OracleUnit(envelope(_numpy_callback(f, caps["a"]), nout))]
    outs = [[], []]
    for j, u in enumerate(us):
        u.set_sample_rate(sr)
        outs[j].append(u.process_many(64 * 30 + 13))
        u.L.fo_set(u.h, P_INTERVAL, (C.c_float * 1)(0.0007), 1, 0, None, 0)
        outs[j].append(u.process_many(64 * 20 + 5))
        outs[j].append(np.stack([u.tick(()) for _ in range(333)], axis=1))
    a, b = (np.concatenate(o, axis=1) for o in outs)
    assert a.shape == (nout, 64 * 50 + 18 + 333) and np.abs(a).max() > 0.1
    assert np.array_equal(a, b), int((a != b).sum())


# ---- 4. NVRTC compiles every class of the GPU file for sm_90a (no GPU needed; into a cache directory of the test's own)
def test_every_gpu_class_compiles_with_nvrtc(tmp_path):
    sigs = sorted({sig(mk(i)) for mk in G.CASES.values() for i in (0, 1)})
    code = ("import sys\nfrom fundsp_b200 import capi\nfor s in sys.stdin.read().split('\\n'):\n"
            "    capi.jit_precompile(s, 1, 1 if ('WaveSynth<' in s or 'PhaseSynth<' in s) else 0)\nprint('compiled', capi.jit_cache_stats())\n")
    env = dict(os.environ, FDSP_JIT_CACHE=str(tmp_path))
    r = subprocess.run([sys.executable, "-c", code], input="\n".join(sigs), capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
    assert r.returncode == 0 and "compiled" in r.stdout, (r.stdout[-500:], r.stderr[-2000:])
    assert len(os.listdir(tmp_path)) >= len(sigs)


# ---- 5. the device node on the host emulation, one voice of every GPU case, against the oracle
@pytest.mark.parametrize("name", sorted(G.CASES))
def test_gpu_case_on_host_emulation(name, tmp_path):
    from test_device_emul_cpu import emulate, oracle
    n = 64 * 40 + 61
    mk = G.CASES[name]
    want = oracle(G.oracle_of(mk(3)), n)
    got, s = emulate(mk(3), n, None, str(tmp_path))
    assert np.abs(want).max() > 1e-3, name
    assert np.array_equal(got, want), (name, int((got != want).sum()), float(np.abs(got - want).max()), s)


# ---- 6. the GPU file on the CPU mock device
def test_gpu_envelope_text_file_on_the_mock_device(mock_env):
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_envelope_text.py"), "-m", "gpu", "-q", "-n", "4",
                        "-p", "no:cacheprovider", "--tb=short"], capture_output=True, text=True, env=mock_env, cwd=ROOT, timeout=1800)
    tail = r.stdout[-3000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail

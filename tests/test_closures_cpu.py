"""Closures of the signal without a GPU: the closure language (accepted and refused texts, with the refusal's token and column), canonical
class signatures, the oracle's closure nodes pinned against built-in nodes and numpy, NVRTC compilation of every closure class of
tests/test_gpu_closures.py for sm_90a, the device templates on the host emulation against the oracle, and the GPU file itself on the
CPU mock device."""
import os
import subprocess
import sys

import numpy as np
import pytest

from fundsp_b200 import capi
from fundsp_b200.capi import FdspError
from fundsp_b200.graph import ArityError
from fundsp_b200.prelude import *  # noqa: F401,F403
from oracle import OracleUnit, lib as olib
import oracle_closure  # noqa: F401  (the oracle's closure nodes, registered on OracleBackend)
from test_mock_bank_cpu import ROOT, mock_env  # noqa: F401  (the mock device build, shared with that file)

import test_gpu_closures as G


def sig(g):
    return capi.NodeHandle(g).signature()


# ---- 1. the language
ACCEPTED = [
    ("|x| x[0]", 1, 1),
    ("move |x: &Frame<f32, U1>| -x[0] * 0.5", 1, 1),
    ("|x| { let a = x[0]; let b: f32 = a * a; (a, b) }", 1, 2),
    ("|x| if x[0] > 0.0 && x[1] <= 1e-3 || !(x[0] != x[1]) { x[0] } else if x[1] < 2. { x[1] } else { 1_000.0f32 }", 2, 1),
    ("|x| (x[1], x[0],)", 2, 2),
    ("|x| x[0].abs().min(x[1]).max(-1.0).clamp(-0.5, 0.5).floor().ceil().round().sqrt().signum()", 2, 1),
    ("|x| x[0].sin() + x[0].cos() + x[0].tan() + x[0].tanh() + x[0].exp() + x[0].powf(2.0)", 1, 1),
    ("|x| abs(x[0]) + min(x[0], 1.0) + max(x[0], 0.0) + clamp(0.0, 1.0, x[0]) + clamp01(x[0]) + clamp11(x[0]) + floor(x[0]) + ceil(x[0])"
     " + round(x[0]) + sqrt(x[0]) + signum(x[0]) + lerp(0.0, 1.0, x[0]) + lerp11(0.0, 1.0, x[0]) + delerp(0.0, 2.0, x[0])"
     " + delerp11(0.0, 2.0, x[0]) + softsign(x[0]) + softexp(x[0]) + smooth3(x[0]) + smooth5(x[0]) + smooth7(x[0]) + smooth9(x[0])"
     " + spline(0.0, 1.0, 0.5, 0.0, x[0]) + sqr_hz(1.0, x[0]) + tri_hz(1.0, x[0]) + bpm_hz(x[0]) + squared(x[0])", 1, 1),
    ("|x| sin(x[0]) + cos(x[0]) + tan(x[0]) + tanh(x[0]) + exp(x[0]) + pow(x[0], 0.5) + exp10(x[0]) + db_amp(x[0]) + sin_hz(1.0, x[0]) + cos_hz(1.0, x[0])", 1, 1),
    ("|x| /* a comment */ x[0] // and another\n * 2.0", 1, 1),
]

# (text, inputs, outputs, exception, the message must contain)
REFUSED = [
    ("|x| x[0] + 2", 1, 1, FdspError, "`2` at column 12: integer literals are not supported"),
    ("|x| x[0] * 0.5f64", 1, 1, FdspError, "`0.5f64` at column 12: only f32 literals"),
    ("|x| log(x[0])", 1, 1, FdspError, "`log` at column 5: its musl source is not restated"),
    ("|x| x[0].log2()", 1, 1, FdspError, "`log2` at column 10: its musl source is not restated"),
    ("|x| xerp(1.0, 2.0, x[0])", 1, 1, FdspError, "`xerp` at column 5: its musl source is not restated"),
    ("|x| atan(x[0]) + exp2(x[0])", 1, 1, FdspError, "`atan` at column 5"),
    ("|x| amp_db(x[0])", 1, 1, FdspError, "`amp_db` at column 5"),
    ("|x| x[0] as f32", 1, 1, FdspError, "`as` at column 10: `as` casts are not supported"),
    ("|x| x[0] % 2.0", 1, 1, FdspError, "`%` at column 10: operator not supported"),
    ("|x| { let mut a = x[0]; a }", 1, 1, FdspError, "`mut` at column 11: mutation is not supported"),
    ("|x| { let a = x[0]; a = 1.0; a }", 1, 1, FdspError, "`=` at column 23: assignment is not supported"),
    ("|x| x[0] += 1.0", 1, 1, FdspError, "`+=` at column 10: assignment is not supported"),
    ("|x| for i in 0..2 { x[0] }", 1, 1, FdspError, "`for` at column 5: loops are not supported"),
    ("|x| foo(x[0])", 1, 1, FdspError, "`foo` at column 5: function not supported"),
    ("|x| x[0].frobnicate()", 1, 1, FdspError, "`frobnicate` at column 10: method not supported"),
    ("|x| x[0] < 1.0 < 2.0", 1, 1, FdspError, "`<` at column 16: comparison operators cannot be chained"),
    ("|x| x[0] + (x[0] > 1.0)", 1, 1, FdspError, "a bool where an f32 is expected"),
    ("|x| if x[0] { 1.0 } else { 0.0 }", 1, 1, FdspError, "an f32 where a bool is expected"),
    ("|x| if x[0] > 0.0 { 1.0 }", 1, 1, FdspError, "an `if` needs an `else`"),
    ("|x| x[0] * k", 1, 1, FdspError, "`k` is neither a parameter nor a captured value"),
    ("|x| x[0] $", 1, 1, FdspError, "`$` at column 10"),
    ("|x| (x[0], 1.0)", 1, 1, ArityError, "arity mismatch: the closure returns 2 values, the node has 1 output"),
    ("|x| x[0]", 1, 2, ArityError, "arity mismatch: the closure returns 1 value, the node has 2 outputs"),
    ("|x, y| x[0]", 1, 1, ArityError, "arity mismatch: map takes one frame parameter"),
    ("|x| x[2]", 2, 1, ArityError, "`2` at column 7: arity mismatch: index 2 of a frame of 2 inputs"),
]


@pytest.mark.parametrize("text,nin,nout", ACCEPTED)
def test_accepted_closure_texts(text, nin, nout):
    h = capi.NodeHandle(map_(text, nin, nout))
    assert h.inputs() == nin and h.outputs() == nout and h.signature().startswith(f"Map<{nin},{nout},0,Ex::")


@pytest.mark.parametrize("text,nin,nout,exc,msg", REFUSED)
def test_refused_closure_texts(text, nin, nout, exc, msg):
    with pytest.raises(exc) as e:
        map_(text, nin, nout)
    assert msg in str(e.value), str(e.value)
    if exc is FdspError:
        assert e.value.code == capi.ERR_ARG


def test_refusals_of_the_other_nodes_and_of_captures():
    with pytest.raises(FdspError, match="capture `k` does not occur in the closure"):
        map_("|x| x[0]", 1, 1, k=1.0)
    with pytest.raises(ArityError, match="shape_fn takes one parameter"):
        shape_fn("|x, y| x")
    with pytest.raises(FdspError, match="only a frame parameter can be indexed"):
        shape_fn("|x| x[0]")
    with pytest.raises(ArityError, match="envelope_in takes"):
        envelope3("|t| t")
    with pytest.raises(ArityError, match="the closure returns 2 values, the node has 1 output"):
        envelope2("|t, x| (t, x)")
    with pytest.raises(FdspError, match="the limit is 4096"):
        map_("|x| " + " + ".join(["x[0]"] * 1200), 1, 1)
    with pytest.raises(FdspError, match="more than 256 operations"):
        map_("|x| " + " + ".join(["x[0]"] * 300), 1, 1)


def test_envelope_parameter_forms():
    assert sig(envelope2("|t, x| t * x")) == sig(envelope_in("|t, i| t * i[0]", 1))
    assert sig(envelope3("|t, x, y| x * y")) == sig(envelope_in("|t, i| i[0] * i[1]", 2))
    assert sig(lfo2("|t, x| x")) == sig(envelope2("|t, x| x")) and sig(lfo3("|t, x, y| y")) == sig(envelope3("|t, x, y| y"))
    assert sig(lfo_in("|t, i| t", 3)) == "EnvelopeInFn<3,1,0,Ex::T>"


# ---- 2. canonical signatures
def test_signatures_are_canonical():
    a = map_("|x| tanh(x[0] * drive)", 1, 1, drive=0.7)
    c = map_("move |frame: &Frame<f32, U1>|   tanh( frame[0]*drive ) // drive it", 1, 1, drive=-3.0)
    assert sig(a) == sig(c) == "Map<1,1,1,Ex::Tanh<Ex::Mul<Ex::In<0>,Ex::Cap<0>>>>"
    assert sig(map_("|x| { let u = x[0]; u * 2.0 }", 1, 1)) == sig(map_("|y| { let w: f32 = y[0]; w * 2.0 }", 1, 1))
    assert sig(map_("|x| x[0] * 0.5", 1, 1)) == sig(map_("|x| x[0] * 5e-1", 1, 1)) == sig(map_("|x| x[0] * 0.5f32", 1, 1))
    assert sig(map_("|x| x[0] * 0.5", 1, 1)) != sig(map_("|x| x[0] * 0.25", 1, 1))
    assert sig(map_("|x| x[0] * k", 1, 1, k=1.0)) != sig(map_("|x| x[0] * 1.0", 1, 1))
    # literals: decimal straight to f32, rounded once
    assert sig(map_("|x| x[0] * 0.1", 1, 1)).endswith(f"Ex::Lit<0x{np.float32(0.1).view(np.uint32):08x}u>>>")
    assert sig(map_("|x| x[0] * 16777217.0", 1, 1)).endswith("Ex::Lit<0x4b800000u>>>")
    # the captured values are per-voice parameter words, in order of first occurrence in the text
    P, _, _ = capi.NodeHandle(map_("|x| x[0] * b + a", 1, 1, a=2.0, b=3.0)).lowering()
    assert list(P.view(np.float32)) == [3.0, 2.0]


def test_one_class_for_sixteen_thousand_voices_on_the_mock_device(mock_env):
    code = ("from fundsp_b200.bank import GpuBank\nfrom fundsp_b200.prelude import map_, saw_hz\n"
            "b = GpuBank([saw_hz(50.0 + 0.05 * i) >> map_('|x| tanh(x[0] * drive)', 1, 1, drive=0.5 + i / 16384.0) for i in range(16384)], per_voice=False, mix=True)\n"
            "print('classes', b.L.fdsp_bank_num_classes(b.h), b.voices())\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=mock_env, cwd=ROOT, timeout=900)
    assert r.returncode == 0 and "classes 1 16384" in r.stdout, (r.stdout[-500:], r.stderr[-1500:])


# ---- 3. oracle pins
def _run(g, n, x=None):
    olib().fo_set_denormal_emulation(0)
    return OracleUnit(g).process_many(n, x)


def test_oracle_closures_equal_builtin_nodes():
    n = 64 * 5 + 13
    x = np.random.default_rng(1).uniform(-3.0, 3.0, (2, n)).astype(np.float32)
    for h in (0.3, 1.0, 2.7):
        assert np.array_equal(_run(shape_fn("|x| tanh(x * h)", h=h), n, x[:1]), _run(shape(Tanh(h)), n, x[:1]))
    assert np.array_equal(_run(map_("|x| x[0] * x[1]", 2, 1), n, x), _run(pass_() * pass_(), n, x))
    assert np.array_equal(_run(map_("|x| (x[1], x[0])", 2, 2), n, x), _run(reverse(2), n, x))
    for c in (0.25, -1.5):
        assert np.array_equal(_run(dc(c) >> envelope2("|t, x| x"), n), _run(dc(c), n))


EXACT = [   # (closure of x[0], x[1]; numpy float32 form)
    ("|x| x[0] * x[1] + 0.5", lambda a, b: a * b + np.float32(0.5)),
    ("|x| min(x[0], x[1]) - max(x[0], 0.25).abs()", lambda a, b: np.fmin(a, b) - np.abs(np.fmax(a, np.float32(0.25)))),
    ("|x| clamp(-0.5, 0.5, x[0]) / (x[1].abs() + 1.0)", lambda a, b: np.fmin(np.fmax(a, np.float32(-0.5)), np.float32(0.5)) / (np.abs(b) + np.float32(1.0))),
    ("|x| if x[0] > x[1] { x[0] - x[1] } else { squared(x[1]) }", lambda a, b: np.where(a > b, a - b, b * b)),
    ("|x| floor(x[0]) + ceil(x[1]) * round(x[0])", lambda a, b: np.floor(a) + np.ceil(b) * np.sign(a) * np.floor(np.abs(a) + np.float32(0.5))),
    ("|x| lerp(x[0], x[1], 0.3)", lambda a, b: a * (np.float32(1.0) - np.float32(0.3)) + b * np.float32(0.3)),
    ("|x| softsign(x[0]) + sqrt(x[1].abs())", lambda a, b: a / (np.float32(1.0) + np.abs(a)) + np.sqrt(np.abs(b))),
    ("|x| { let d = x[0] - x[1]; d * d * -2.0 }", lambda a, b: (a - b) * (a - b) * np.float32(-2.0)),
]


@pytest.mark.parametrize("k", range(len(EXACT)))
def test_oracle_exact_operations_against_numpy(k):
    text, f = EXACT[k]
    n = 64 * 4 + 5
    x = np.random.default_rng(k).uniform(-4.0, 4.0, (2, n)).astype(np.float32)
    with np.errstate(all="ignore"):
        want = f(x[0], x[1]).astype(np.float32)
    got = _run(map_(text, 2, 1), n, x)[0]
    assert np.array_equal(got, want), (text, int((got != want).sum()))


def test_reference_envelope2_envelope3_lines():
    """tests/test_basic.rs:177-181 of the reference, in prelude32 form: lfo2 / envelope2(|t, x| t * x) on dc(1.0), lfo3 / envelope3(|t, x, y|
    t * x * y) on dc((1.0, 2.0)); check_wave requires tick and process to agree within 1e-4."""
    n = 64 * 20 + 17
    for g in (dc(1.0) >> lfo2("|t, x| t * x") | dc(1.0) >> envelope2("|t, x| t * x"),
              dc((1.0, 2.0)) >> lfo3("|t, x, y| t * x * y") | dc((1.0, 2.0)) >> envelope3("|t, x, y| t * x * y")):
        olib().fo_set_denormal_emulation(0)
        proc = OracleUnit(g).process_many(n)
        u = OracleUnit(g)
        tick = np.stack([u.tick(()) for _ in range(n)], axis=1)
        assert np.abs(proc).max() > 0.01 and np.abs(proc - tick).max() <= 1e-4


# ---- 4. NVRTC compiles every closure class of the GPU file for sm_90a (no GPU needed; into a cache directory of the test's own)
def test_every_gpu_closure_class_compiles_with_nvrtc(tmp_path):
    sigs = sorted({sig(mk(i)) for mk in G.CASES.values() for i in (0, 1)})
    code = ("import sys\nfrom fundsp_b200 import capi\nfor s in sys.stdin.read().split('\\n'):\n"
            "    capi.jit_precompile(s, 1, 1 if ('WaveSynth<' in s or 'PhaseSynth<' in s) else 0)\nprint('compiled', capi.jit_cache_stats())\n")
    env = dict(os.environ, FDSP_JIT_CACHE=str(tmp_path))
    r = subprocess.run([sys.executable, "-c", code], input="\n".join(sigs), capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
    assert r.returncode == 0 and "compiled" in r.stdout, (r.stdout[-500:], r.stderr[-2000:])
    assert len(os.listdir(tmp_path)) >= len(sigs)


# ---- 5. the device templates on the host emulation, one voice of every GPU case, against the oracle
@pytest.mark.parametrize("name", sorted(G.CASES))
def test_gpu_case_on_host_emulation(name, tmp_path):
    from test_device_emul_cpu import emulate, oracle
    n = 64 * 40 + 61
    mk = G.CASES[name]
    want = oracle(mk(3), n)
    got, s = emulate(mk(3), n, None, str(tmp_path))
    assert np.abs(want).max() > 1e-3, name
    assert np.array_equal(got, want), (name, int((got != want).sum()), float(np.abs(got - want).max()), s)


# ---- 6. the GPU file on the CPU mock device
def test_gpu_closure_file_on_the_mock_device(mock_env):
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_closures.py"), "-m", "gpu", "-q", "-n", "4",
                        "-p", "no:cacheprovider", "--tb=short"], capture_output=True, text=True, env=mock_env, cwd=ROOT, timeout=1800)
    tail = r.stdout[-3000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail

"""`update` without a GPU: the update closure form (accepted and refused texts, with their columns), canonical signatures and one class
for voices that differ in captures or dt, the word layout with the set values in state, the inner hashes after System's re-ping against
the oracle's, the oracle's System against a Python model of src/system.rs, every case of tests/test_gpu_update.py on the host emulation
and through NVRTC for sm_90a, and that GPU file on the CPU mock device."""
import ctypes as C
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
from test_mock_bank_cpu import ROOT, mock_env  # noqa: F401  (the mock device build, shared with that file)
from update_oracle import oracle_of, split_update

import test_gpu_update as G

F32 = np.float32
VOICE = lambda: saw_hz(110.0) >> lowpass_hz(1000.0, 1.0)


def sig(g):
    return capi.NodeHandle(g).signature()


# ---- 1. the language
ACCEPTED = [
    "|t, dt, x| x.set(Setting::center(t).right())",
    "move |t: f32, dt: f32, x: &mut An<X>| { x.set(Setting::center_q(t, dt).index(1)); }",
    "|time, delta, node| { let a = time * 2.0; let b = if a < 1.0 { a } else { 1.0 }; node.set(Setting::center_q_gain(a, b, 1.0).right()); node.set(Setting::value(delta).left().left()) }",
    "|t, dt, x| { x.set(Setting::pan(sin_hz(1.0, t))); x.set(Setting::biquad(0.1, 0.2, 0.3, 0.4, 0.5)) }",
]

REFUSED = [   # (text, exception, the message must contain)
    ("|t, dt| t", ArityError, "update: arity mismatch: update takes |t, dt, x|, the text has 2 parameters"),
    ("|t, dt, x| if t < 1.0 { x.set(Setting::center(1.0)) } else { x.set(Setting::center(2.0)) }", FdspError,
     "`if` at column 12: a `set` inside an `if` is not supported"),
    ("|t, dt, x| x.set(Setting::center(x))", FdspError, "`x` at column 34: the node parameter can only be the receiver of `.set(..)`"),
    ("|t, dt, x| x.set(Setting::center(1.0).node(2))", FdspError, "`node` at column 39: `.node()` addressing is not supported"),
    ("|t, dt, x| x.set(Setting::delay(1.0))", FdspError, "`delay` at column 27: setting not supported in an update function"),
    ("|t, dt, x| { let a = t; }", FdspError, "`}` at column 25: the update function sets nothing"),
    ("|t, dt, x| x.reset()", FdspError, "`reset` at column 14: only `.set(..)` can be called on the node parameter"),
    ("|t, dt, x| x.set(Setting::center(1.0, 2.0))", FdspError, "`center` at column 27: takes 1 argument, given 2"),
    ("|t, dt, x| x.set(Setting::center(1.0).index(1.0))", FdspError, "`1.0` at column 45: `.index()` takes an integer literal"),
    ("|t, dt, x| { x.set(Setting::center(1.0)); let a = t; }", FdspError, "`let` at column 43: a `let` after a `set` is not supported"),
    ("|t, dt, x| x.set(Setting::center(t * 2))", FdspError, "`2` at column 38: integer literals are not supported"),
    ("|t, dt, x| x.set(Setting::center(log(t)))", FdspError, "`log` at column 34: its musl source is not restated"),
    ("|t, dt, x| x.set(Setting::center(t)) x.set(Setting::center(t))", FdspError, "`x` at column 38: expected `;`"),
]


@pytest.mark.parametrize("text", ACCEPTED)
def test_accepted_texts(text):
    h = capi.NodeHandle(update(dc(1.0) >> lowpass_hz(1000.0, 1.0) >> pan(0.0), 0.002, text))
    assert h.signature().startswith("System<") and capi.lib().fdsp_node_id(h.h) == 67


@pytest.mark.parametrize("text,exc,msg", REFUSED)
def test_refused_texts(text, exc, msg):
    with pytest.raises(exc) as e:
        update(VOICE(), 0.002, text)
    assert msg in str(e.value), str(e.value)
    if exc is FdspError:
        assert e.value.code == capi.ERR_ARG


def test_refusals_of_captures_and_callables():
    with pytest.raises(FdspError, match="update: capture `k` does not occur in the closure"):
        update(VOICE(), 0.002, "|t, dt, x| x.set(Setting::center(t))", k=1.0)
    with pytest.raises(FdspError, match="`r` is neither a parameter nor a captured value"):
        update(VOICE(), 0.002, "|t, dt, x| x.set(Setting::center(r))")
    with pytest.raises(TypeError, match="update takes its function as text"):
        update(VOICE(), 0.002, lambda t, dt, x: None)
    lib = capi.lib()
    assert not lib.fdsp_update(None, 0.002, b"|t, dt, x| x.set(Setting::center(t))", 0, None, None)
    assert b"update: null node" in lib.fdsp_last_error()


# ---- 2. canonical signatures; captures and dt are per-voice words
def test_signatures_are_canonical_and_one_class():
    a = update(VOICE(), 0.002, G.SWEEP, r=0.5)
    b = update(VOICE(), 0.01, "move |time: f32, d, node|   node.set( Setting::center(600.0 + 400.0*sin_hz(r,time)).right() ); // sweep", r=3.0)
    assert sig(a) == sig(b) == ("System<Pipe<Pipe<Constant<1>,WaveSynth<0,1>>,FixedSvf>,3,1,Ex::Out<Ex::Add<Ex::Lit<0x44160000u>,Ex::Mul<Ex::Lit<0x43c80000u>,"
                                "Ex::SinHz<Ex::Cap<0>,Ex::In<0>>>>>,UpdTargets<UpdTarget<0,0,0,0,-1,-1,-1,-1,UpdAt<1>>>>")
    assert sig(update(VOICE(), 0.002, G.SWEEP.replace(".right()", ".left()"), r=0.5)).endswith("UpdTargets<>>")   # the saw ignores it
    assert sig(a) != sig(update(VOICE(), 0.002, G.SWEEP.replace("center(", "center_q(1.0, "), r=0.5))
    # the last statement that writes a value gives it; the q of center_q, the gain of center_q_gain
    s = sig(update(VOICE(), 0.002, "|t, dt, x| { x.set(Setting::center_q_gain(t, dt, 2.0).right()); x.set(Setting::center(dt).right()) }"))
    assert s.endswith("Ex::Out<Ex::In<0>,Ex::In<1>,Ex::Lit<0x40000000u>,Ex::In<1>>,UpdTargets<UpdTarget<0,0,0,3,1,2,-1,-1,UpdAt<1>>>>"), s


def test_settings_the_reached_node_ignores_are_ignored():
    """A Resonator has no set() in the reference, so no statement makes it a target; a `center` reaching the saw is ignored like the
    saw's own set() ignores it, not refused; one reaching a Moog, which takes it, is refused when the bank is built."""
    reson = sig(update(saw_hz(110.0) >> resonator_hz(500.0, 50.0), 0.002, "|t, dt, x| { x.set(Setting::center_q(t, 2.0).right()); x.set(Setting::center(t).right()) }"))
    assert reson.endswith("UpdTargets<>>"), reson
    P, S, _ = capi.NodeHandle(update(saw_hz(110.0) >> resonator_hz(500.0, 50.0), 0.002, "|t, dt, x| x.set(Setting::center(t).right())")).lowering()
    assert len(S) == 2 + len(capi.NodeHandle(saw_hz(110.0) >> resonator_hz(500.0, 50.0)).lowering()[1])   # time, delta_time and no set values
    audio_rate = sig(update((saw_hz(110.0) | dc(1000.0) | dc(1.0)) >> lowpass(), 0.002, "|t, dt, x| x.set(Setting::center(t).right())"))
    assert audio_rate.endswith("UpdTargets<>>"), audio_rate   # Svf (ID 36) has no set() in the reference
    osc = sig(update(VOICE(), 0.002, "|t, dt, x| { x.set(Setting::center(t).left().right()); x.set(Setting::center(t).right()) }"))
    assert osc.endswith("UpdTargets<UpdTarget<0,0,0,1,-1,-1,-1,-1,UpdAt<1>>>>"), osc


def test_word_layout_with_set_values_in_state():
    g = update(saw_hz(110.0) >> (butterpass_hz(700.0) >> lowpass_hz(1200.0, 2.0)), 0.004,
               "|t, dt, x| { x.set(Setting::center_q(a * t, 1.5).right().right()); x.set(Setting::center(b).right().left()) }", a=3.0, b=5.0)
    P, S, U = capi.NodeHandle(g).lowering()
    inner_P, inner_S, _ = capi.NodeHandle(saw_hz(110.0) >> (butterpass_hz(700.0) >> lowpass_hz(1200.0, 2.0))).lowering()
    assert list(P.view(F32)[:3]) == [F32(0.004), 3.0, 5.0] and list(P[3:]) == list(inner_P)
    # time, delta_time, then the targets in order of first statement: the SVF's (cutoff, q, gain), the ButterLowpass's cutoff
    assert list(S.view(F32)[:6]) == [0.0, 0.0, 1200.0, 2.0, 1.0, 700.0] and len(S) == 6 + len(inner_S) and len(U) == 0   # (the saw's phase follows the re-ping)


# ---- 3. System re-pings its inner node from AttoHash::new(67): the inner hashes differ from the bare node's and equal the oracle's
def test_inner_hashes_after_the_reping():
    bare = lambda: noise() >> lowpass_hz(1000.0, 1.0) | sine_hz(3.0)
    mk = lambda: update(bare(), 0.002, "|t, dt, x| x.set(Setting::center(t).left().right())")
    want = OracleUnit(oracle_of(mk())).leaf_hashes()
    assert want != OracleUnit(bare()).leaf_hashes()
    assert capi.NodeHandle(mk()).leaf_hashes() == want
    assert capi.NodeHandle(bare()).leaf_hashes() == OracleUnit(bare()).leaf_hashes()


# ---- 4. the oracle's System against a Python model of src/system.rs at ragged block sizes, size 0 and dt = 0
def _model(sizes, sr, dt):
    """The (t, dt) of the last update System::process has made after each nonempty block of `sizes`, in f32."""
    time = delta = F32(0.0)
    cur, out = None, []
    for size in sizes:
        delta_now = F32(F32(size) / F32(sr))
        if delta >= F32(dt) or (time == 0.0 and size > 0):
            cur = (time, delta)
            delta = F32(0.0)
        time = F32(time + delta_now)
        delta = F32(delta + delta_now)
        if size:
            out.append(cur)
    return out


@pytest.mark.parametrize("dt", [0.0, 0.0005, 64.0 / 48000.0, 0.003])
def test_oracle_system_against_a_model(dt):
    olib().fo_set_denormal_emulation(0)
    sizes = [64, 0, 1, 7, 63, 64, 0, 0, 33, 8, 64, 64, 2, 40, 64, 5] * 6
    # the first constant takes the t of each update, the second its dt: a block's output shows the last update made up to it
    g = update(dc(-1.0) | dc(-1.0), dt, "|t, dt, x| { x.set(Setting::value(t).left()); x.set(Setting::value(dt).right()) }")
    u = OracleUnit(oracle_of(g))
    u.set_sample_rate(48000.0)
    seen = [(F32(o[0, 0]), F32(o[1, 0])) for o in (u.process(size) for size in sizes) if o.shape[1]]
    want = _model(sizes, 48000.0, dt)
    assert seen == want and len(set(want)) > 10


# ---- 5. every GPU case on the host emulation, bit for bit against the oracle
@pytest.mark.parametrize("name", sorted(G.CASES))
def test_gpu_case_on_host_emulation(name, tmp_path):
    from test_device_emul_cpu import emulate, oracle
    n = 64 * 40 + 61
    mk = G.CASES[name]
    want = oracle(G.expected(name, 3), n)
    got, s = emulate(mk(3), n, None, str(tmp_path))
    assert np.abs(want).max() > 1e-3, name
    assert np.array_equal(got, want), (name, int((got != want).sum()), float(np.abs(got - want).max()), s)


# ---- 6. NVRTC compiles every class of the GPU file for sm_90a (no GPU needed; into a cache directory of the test's own)
def test_every_gpu_class_compiles_with_nvrtc(tmp_path):
    sigs = sorted({sig(mk(i)) for mk in G.CASES.values() for i in (0, 1)})
    code = ("import sys\nfrom fundsp_b200 import capi\nfor s in sys.stdin.read().split('\\n'):\n"
            "    capi.jit_precompile(s, 1, 1 if ('WaveSynth<' in s or 'PhaseSynth<' in s) else 0)\nprint('compiled', capi.jit_cache_stats())\n")
    env = dict(os.environ, FDSP_JIT_CACHE=str(tmp_path))
    r = subprocess.run([sys.executable, "-c", code], input="\n".join(sigs), capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
    assert r.returncode == 0 and "compiled" in r.stdout, (r.stdout[-500:], r.stderr[-2000:])
    assert len(os.listdir(tmp_path)) >= len(sigs)


# ---- 7. the GPU file on the CPU mock device
def test_gpu_update_file_on_the_mock_device(mock_env):
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_update.py"), "-m", "gpu", "-q", "-n", "4",
                        "-p", "no:cacheprovider", "--tb=short"], capture_output=True, text=True, env=mock_env, cwd=ROOT, timeout=1800)
    tail = r.stdout[-3000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail


def test_split_update_reads_the_statements():
    assert split_update(G.SWEEP_QG) == ("t", "dt", ["let u = tri_hz(r, t);"], [(3, ["900.0 + 600.0 * u", "0.8 + 0.2 * u", "1.0 + u"], [1])])

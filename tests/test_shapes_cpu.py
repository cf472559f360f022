"""The Atan and Adaptive waveshapes without a GPU: the product's atanf_ / wide_atanf against the oracle's restatements bit for bit and
against float64, known answers of both shapes, the reference's nonlinear-biquad lines with Atan, the C ABI's refusals, NVRTC
compilation of every class of tests/test_gpu_shapes.py for sm_90a, the device templates on the host emulation against the oracle, and
the GPU file itself on the CPU mock device."""
import os
import subprocess
import sys

import numpy as np
import pytest

from fundsp_b200 import capi
from fundsp_b200.capi import FdspError
from fundsp_b200.prelude import *  # noqa: F401,F403
from oracle import OracleUnit, lib as olib
import oracle_shapes
from test_mock_bank_cpu import ROOT, mock_env  # noqa: F401  (the mock device build, shared with that file)

import test_gpu_shapes as G

F32 = np.float32


def sig(g):
    return capi.NodeHandle(g).signature()


# ---- 1. scalar math: every 97th float pattern here; `libm_equiv_atan 1` walks all 2^32 (both bit-identical; max 0.852 ulp for atanf,
# 2.849 ulp for wide_atanf, the bar below)
def test_product_atan_equals_oracle_and_float64(tmp_path):
    exe = str(tmp_path / "libm_equiv_atan")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-pthread", "-w", os.path.join(ROOT, "tests", "cpp", "libm_equiv_atan.cpp"), "-o", exe])
    r = subprocess.run([exe, "97"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.count("bit-identical") == 2, r.stdout
    ulp = {ln.split(":")[0]: float(ln.split("max ulp ")[1].split()[0]) for ln in r.stdout.splitlines() if "max ulp" in ln}
    assert ulp["atanf"] <= 1.0 and ulp["wide_atanf"] <= 3.0, ulp


def test_oracle_atanf_against_numpy():
    L = oracle_shapes.lib()
    x = np.concatenate([np.linspace(-30.0, 30.0, 20001), np.geomspace(1e-8, 1e12, 2001)]).astype(F32)
    got = np.array([L.fo_atanf(float(v)) for v in x], F32)
    exact = np.arctan(x.astype(np.float64))
    spacing = np.spacing(np.abs(exact.astype(F32))).astype(np.float64)
    assert (np.abs(got - exact) / spacing).max() <= 1.0


# ---- 2. known answers
def _ticks(g, xs, reset=False):
    olib().fo_set_denormal_emulation(0)
    u = OracleUnit(g)
    if reset:
        u.reset()
    return np.array([u.tick((float(v),))[0] for v in xs], F32)


def test_atan_known_answers():
    x = np.float32([-1e30, -5.0, -1.0, -0.3, -1e-4, 0.0, 1e-4, 0.3, 1.0, 5.0, 1e30])
    for h in (0.25, 1.0, 3.0):
        y = _ticks(shape(Atan(h)), x)
        assert np.array_equal(y, -y[::-1]), h                          # odd
        assert np.abs(y).max() <= 1.0                                  # saturates at unity
    y = _ticks(shape(Atan(1.0)), np.float32([1e-4, 1e-6]))
    assert np.allclose(y / np.float32([1e-4, 1e-6]), 1.0, rtol=1e-6)   # slope 1 at the origin for h = 1
    inf = _ticks(shape(Atan(1.0)), np.float32([np.inf, -np.inf]))
    want = np.uint32(0x3fc90fda).view(F32) * (F32(2.0) / F32(np.pi))   # atanf(inf) = atan(inf)hi + 2^-120, times 2 / PI in f32
    assert inf.view(np.uint32).tolist() == [want.view(np.uint32), (-want).view(np.uint32)]


def test_atan_parameter_word_is_folded_in_f32():
    for h in (0.3, 1.0, 7.5):
        P, S, U = capi.NodeHandle(shape(Atan(h))).lowering()
        assert P.view(F32)[0] == F32(h) * F32(np.pi) * F32(0.5) and len(S) == 0


def test_reference_nonlinear_biquad_lines_with_atan():
    """tests/test_basic.rs:226-233 of the reference as written: check_wave requires tick and process to agree within 1e-4."""
    n, sr = 441, 44100.0
    for g in (noise() >> fbell_hz(Atan(1.0), 500.0, 50.0, 0.5) | noise() >> flowpass_hz(Clip(1.0), 2000.0, 2.0),
              noise() >> fresonator_hz(Atan(0.5), 500.0, 50.0) | noise() >> fhighpass_hz(Softsign(0.2), 2000.0, 2.0),
              noise() >> shape(Atan(2.0)) | noise().seed(2) >> shape(Atan(0.5))):   # and the block path's wide atan
        olib().fo_set_denormal_emulation(0)
        a = OracleUnit(g)
        wave = a.render(sr, n / sr)
        a.reset()
        ticks = np.stack([a.tick() for _ in range(n)], axis=1)
        assert np.abs(wave).max() > 1e-3 and np.abs(wave - ticks).max() <= 1e-4


def _smoothing(g, sr=None):
    h = capi.NodeHandle(g)
    if sr:
        h.set_sample_rate(sr)
    return float(h.lowering()[0].view(F32)[0])


def test_adaptive_known_answers():
    ts, x0 = 0.01, F32(0.5)
    sm = F32(_smoothing(shape(Adaptive(ts, Tanh(1.0)))))
    assert abs(float(sm) ** (ts * 44100.0) - 0.5) < 1e-4
    assert abs(_smoothing(shape(Adaptive(ts, Tanh(1.0))), 48000.0) ** (ts * 48000.0) - 0.5) < 1e-4
    # inside a biquad the smoothing keeps Adaptive::new's 44.1 kHz value at any rate
    assert _smoothing(flowpass_hz(Adaptive(ts, Tanh(1.0)), 500.0, 2.0), 48000.0) == float(sm)
    # the first sample from the state of a new unit (0.0) and of a reset one (1e-3)
    for reset, st in ((False, F32(0.0)), (True, F32(1e-3))):
        level = sm * st + (F32(1.0) - sm) * (F32(1e-6) + x0 * x0)
        want = np.tanh(np.float64(x0 / np.sqrt(level)))
        got = _ticks(shape(Adaptive(ts, Tanh(1.0))), [x0], reset)[0]
        assert abs(float(got) - want) <= 2e-7, (reset, got, want)
        got = _ticks(shape(Adaptive(ts, ClipTo(-1e9, 1e9))), [x0], reset)[0]
        assert got == x0 / np.sqrt(level), reset


@pytest.mark.parametrize("amplitude", [0.01, 1.0, 100.0])
def test_adaptive_normalises_the_level(amplitude):
    """With an identity inner shape the output is the input over its running RMS: sines of any amplitude come out at RMS 1."""
    olib().fo_set_denormal_emulation(0)
    u = OracleUnit(sine_hz(440.0) * dc(amplitude) >> shape(Adaptive(0.01, ClipTo(-1e9, 1e9))))
    y = u.render(44100.0, 1.0)[0]
    rms = float(np.sqrt(np.mean(np.float64(y[22050:]) ** 2)))
    assert abs(rms - 1.0) < 0.02, rms


# ---- 3. refusals and signatures
def test_refusals_and_signatures():
    with pytest.raises(FdspError):
        capi.NodeHandle(An("shaper", (9, 1.0, 0.0), (), 1, 1))
    with pytest.raises(FdspError, match="inner shape must be one of the kinds"):
        capi.NodeHandle(An("shaper_adaptive", (0.01, 7, 1.0, 0.0), (), 1, 1))
    with pytest.raises(FdspError, match="timescale must be a positive"):
        capi.NodeHandle(An("shaper_adaptive", (0.0, 2, 1.0, 0.0), (), 1, 1))
    with pytest.raises(ValueError, match="inner shape must be one of"):
        Adaptive(0.01, Adaptive(0.01, Tanh(1.0)))
    with pytest.raises(ValueError, match="inner shape must be one of"):
        Adaptive(0.01, shape_fn("|x| x * 2.0"))
    assert sig(shape(Atan(2.0))) == sig(shape(Atan(0.1))) == "Shaper<6>"
    assert sig(shape(Adaptive(0.01, Atan(1.0)))) == sig(shape(Adaptive(0.5, Atan(3.0)))) == "ShaperAdaptive<6>"
    assert sig(dbell_hz(Atan(1.0), 1000.0, 2.0, 2.0)) == "NlBiquad<0,3,6,1>"
    assert sig(fresonator(Adaptive(0.01, Crush(4.0)))) == "NlBiquadAdaptive<1,0,4,3>"
    # words: smoothing, p0, p1, then the biquad's own, then one level estimate (FbBiquad) or two (DirtyBiquad), 0.0 in a new unit
    for g, ns in ((shape(Adaptive(0.01, Tanh(2.0))), 1), (flowpass_hz(Adaptive(0.01, Tanh(2.0)), 500.0, 2.0), 3), (dlowpass_hz(Adaptive(0.01, Tanh(2.0)), 500.0, 2.0), 4)):
        P, S, _ = capi.NodeHandle(g).lowering()
        assert P.view(F32)[1:3].tolist() == [2.0, 0.0] and len(S) == ns and not S.any()


# ---- 4. NVRTC compiles every class of the GPU file for sm_90a (no GPU needed; into a cache directory of the test's own)
def test_every_gpu_shape_class_compiles_with_nvrtc(tmp_path):
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
def test_gpu_shape_file_on_the_mock_device(mock_env):
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_shapes.py"), "-m", "gpu", "-q", "-n", "4",
                        "-p", "no:cacheprovider", "--tb=short"], capture_output=True, text=True, env=mock_env, cwd=ROOT, timeout=1800)
    tail = r.stdout[-3000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail

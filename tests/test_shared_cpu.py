"""Shared controls without a GPU: the C ABI and its word layouts, ping hashes against the oracle (IDs 68, 56, 57), the cell's reference
counting, the oracle's Shared nodes pinned by known answers, NVRTC compilation of every writer class, the device templates on the host
emulation against the oracle, and tests/test_gpu_shared.py on the CPU mock device (refusals included)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from fundsp_b200 import capi
from fundsp_b200.graph import ArityError
from fundsp_b200.prelude import *  # noqa: F401,F403
from oracle import OracleUnit, lib as olib
from oracle_shared import mirror
from test_mock_bank_cpu import ROOT, mock_env  # noqa: F401  (the mock device build, shared with that file)

SR = 48000.0
f2u = lambda x: int(np.float32(x).view(np.uint32))


def words64(d):
    u = int(np.float64(d).view(np.uint64))
    return [u & 0xFFFFFFFF, u >> 32]


def test_abi_symbols_and_signatures():
    names = {"fdsp_shared_new", "fdsp_shared_wrap", "fdsp_shared_free", "fdsp_shared_set", "fdsp_shared_get", "fdsp_var_shared",
             "fdsp_monitor_shared", "fdsp_timer"}
    assert names <= set(capi.header_symbols())
    L = capi.lib()
    for n in names:
        assert hasattr(L, n)
    assert L.fdsp_shared_get.restype is C.c_float and L.fdsp_monitor_shared.argtypes == [C.c_void_p, C.c_int, C.c_double]


def test_cell_set_get_wrap_and_references():
    L = capi.lib()
    s = shared(0.25)
    assert s.value() == 0.25
    s.set(1.0 / 3.0)
    assert s.value() == float(np.float32(1.0 / 3.0))
    word = (C.c_uint32 * 1)(f2u(-2.5))                 # memory the caller owns (a Rust AtomicU32)
    released = []
    REL = C.CFUNCTYPE(None, C.c_void_p)
    rel = REL(lambda user: released.append(user))
    L.fdsp_shared_wrap.argtypes = [C.POINTER(C.c_uint32), REL, C.c_void_p]
    h = L.fdsp_shared_wrap(word, rel, 1234)
    assert L.fdsp_shared_get(h) == -2.5
    L.fdsp_shared_set(h, 4.0)
    assert word[0] == f2u(4.0)
    n = L.fdsp_var_shared(h)
    L.fdsp_shared_free(h)                                # the node keeps its own reference
    P = np.zeros(4, np.uint32)
    cnt = [C.c_int(0) for _ in range(3)]
    capi.check(L.fdsp_node_lowering(n, P.ctypes.data_as(C.POINTER(C.c_uint32)), 4, None, 0, None, 0, *[C.byref(c) for c in cnt]))
    assert cnt[0].value == 1 and P[0] == f2u(4.0)
    assert released == []                                # the node still holds the cell
    L.fdsp_node_free(n)
    assert released == [1234]                            # the last reference went: the owner may free the memory
    assert not L.fdsp_var_shared(None) and not L.fdsp_monitor_shared(s.handle, 3, 0.1) and not L.fdsp_monitor_shared(s.handle, 1, 0.0)


def test_word_layouts_and_signatures():
    s = shared(0.75)
    h = capi.NodeHandle(var(s))
    P, S, U = h.lowering()
    assert h.signature() == "Constant<1>" and list(P) == [f2u(0.75)] and len(S) == 0 and len(U) == 0
    for k, m in enumerate((Meter.Sample, Meter.Peak(0.02), Meter.Rms(0.05))):
        h = capi.NodeHandle(monitor(s, m))
        h.set_sample_rate(SR)
        P, S, U = h.lowering()
        sm = 0.0 if k == 0 else float(np.float32(0.5 ** (1.0 / (m[1] * SR))))
        assert h.signature() == f"MonitorShared<{k}>" and list(P) == [f2u(sm)] and list(S) == [0, 0]
    t = shared(3.0)
    h = capi.NodeHandle(timer(t))
    assert t.value() == 0.0                              # Timer::new stores 0
    h.set_sample_rate(SR)
    P, S, U = h.lowering()
    assert h.signature() == "TimerShared" and list(P) == words64(1.0 / SR) and list(S) == [0, 0, 0]
    h = capi.NodeHandle(var_fn(s, "|x| (x * g, x)", 2, g=2.0))
    P, S, U = h.lowering()
    assert h.signature().startswith("VarFn<2,1,") and list(P) == [f2u(0.75), f2u(2.0)] and len(S) == 0
    with pytest.raises(ArityError):
        var_fn(s, "|x| (x, x)", 3)
    with pytest.raises(ArityError):
        var_fn(s, "|x, y| x")
    assert capi.NodeHandle(monitor()).signature() == "MultiPass<1>"   # without a Shared: the plain pass-through, as before


def test_ping_hashes_and_ids_match_the_oracle():
    a, b = shared(0.5), shared(0.0)
    g = (var(a) * saw_hz(220.0) >> monitor(b, Meter.Rms(0.1)) >> lowpass_hz(1000.0, 1.0)) | timer(shared()) | var(a) >> follow(0.01)
    # (the oracle's Shared nodes live in a library of their own, whose leaves its leaf-hash trace does not see: compare the ping chains,
    # and the hashes of the leaves the oracle traces, which follow the Shared leaves)
    for x in (g, var(a), monitor(b, Meter.Peak(0.1)), timer(b) | dc(1.0), var(a) * saw_hz(220.0), var_fn(a, "|x| (x, -x)", 2) | saw_hz(3.0)):
        for probe in (True, False):
            assert capi.NodeHandle(x).ping(probe, 12345) == OracleUnit(x).ping(probe, 12345)
    saw_leaf = lambda x: x.leaf_hashes()[-1]
    assert saw_leaf(capi.NodeHandle(var(a) * saw_hz(220.0))) == saw_leaf(OracleUnit(var(a) * saw_hz(220.0)))
    assert capi.NodeHandle(var(a)).leaf_hashes() == capi.NodeHandle(var(0.5)).leaf_hashes()
    L = capi.lib()
    for node, want in ((var(a), 68), (var_fn(a, "|x| x"), 70), (monitor(b, Meter.Sample), 56), (timer(b), 57)):
        h = capi.NodeHandle(node)
        assert L.fdsp_node_id(h.h) == want


def test_oracle_known_answers():
    olib().fo_set_denormal_emulation(0)
    t = shared(2.0)
    u = OracleUnit(timer(t) | dc(0.0))
    u.set_sample_rate(SR)
    exact = np.float64(0.0)
    for n in range(1, 6):                                # src/shared.rs:230-233: time += size * sample_duration per block, stored as f32
        u.process(64)
        exact += 64.0 * (1.0 / SR)
        assert mirror(t).value() == float(np.float32(exact))
    u.reset()
    assert mirror(t).value() == 0.0
    x = (np.sin(np.arange(64 * 7 + 5) * 0.37) * 0.8).astype(np.float32)
    for m in (Meter.Sample, Meter.Peak(0.01), Meter.Rms(0.02)):
        s = shared(0.0)
        mon, met = OracleUnit(monitor(s, m)), OracleUnit(meter(m))
        for w in (mon, met):
            w.set_sample_rate(SR)
        y = mon.process_many(len(x), x[None])
        lv = met.process_many(len(x), x[None])
        assert np.array_equal(y[0], x)                   # the audio passes through
        want = x[-1] if m[0] == 0 else lv[0, -1]         # Sample: the last input; Peak / Rms: what meter() outputs last
        assert mirror(s).value() == float(want), m


def test_oracle_var_follows_its_cell():
    s = shared(0.5)
    u = OracleUnit(var(s))
    mirror(s).set(0.125)
    assert u.process(10)[0].tolist() == [0.125] * 10


# ---- NVRTC compiles every writer class for sm_90a (no GPU needed; into a cache directory of the test's own)
def test_writer_classes_compile_with_nvrtc(tmp_path):
    s = shared()
    sigs = sorted({capi.NodeHandle(g).signature() for g in
                   [noise() >> monitor(s, m) >> lowpass_hz(500.0, 1.0) for m in (Meter.Sample, Meter.Peak(0.1), Meter.Rms(0.1))] +
                   [timer(s) | saw_hz(100.0), (noise() >> monitor(s, Meter.Sample)) | timer(s),
                    var_fn(s, "|x| (x * g, tanh(x))", 2, g=0.5), var_fn(s, "|x| x * x")]})
    code = ("import sys\nfrom fundsp_b200 import capi\nfor s in sys.stdin.read().split('\\n'):\n"
            "    capi.jit_precompile(s, 1, 1 if ('WaveSynth<' in s or 'PhaseSynth<' in s) else 0)\nprint('compiled', capi.jit_cache_stats())\n")
    env = dict(os.environ, FDSP_JIT_CACHE=str(tmp_path))
    r = subprocess.run([sys.executable, "-c", code], input="\n".join(sigs), capture_output=True, text=True, env=env, cwd=ROOT, timeout=1800)
    assert r.returncode == 0 and "compiled" in r.stdout, (r.stdout[-500:], r.stderr[-2000:])


# ---- the device templates on the host emulation, one voice of every GPU case, against the oracle (a reader's word is the cell's value
# when the voice is lowered)
import test_gpu_shared as G  # noqa: E402
from fundsp_b200.net import Net  # noqa: E402
from fundsp_b200.sequencer import event, slot  # noqa: E402

EMUL = {
    "two_shareds_saw_lowpass": lambda s: G.saw_voice(s, 5),
    "keys_var_follow_cutoff": lambda s: (saw_hz(55.0) | var(s) >> follow(0.01) | dc(1.0)) >> lowpass(),
    "var_fn_tuple": lambda s: (var_fn(s, "|x| { let y = x * g; (y, tanh(y) - x.abs().sqrt()) }", 2, g=1.3) | saw_hz(93.0)) >> (pass_() * pass_() | pass_()),
    "rate_reset_reader_monitor_timer": lambda s: (var(s) * saw_hz(157.0) >> monitor(shared(), Meter.Rms(0.01)) >> lowpass_hz(800.0, 1.0)) | timer(shared()),
    "timer_alone": lambda s: timer(shared()) | saw_hz(77.0),
    "net_reader": lambda s: ((Net.wrap(var(s)) | Net.wrap(saw_hz(103.0))) >> Net.wrap(pass_() * pass_())).node(),
    "event_reader": lambda s: event(var(s) * saw_hz(203.0), 100.0 / G.SR, 2100.0 / G.SR, 1, 40.0 / G.SR, 100.0 / G.SR),
    "slot_reader": lambda s: slot(var(s) * noise().seed(3)),
}
for _k, _m in enumerate(G.METERS):
    EMUL[f"monitor_timer_mode{_k}"] = lambda s, _k=_k: ((noise().seed(3) * 0.5 >> monitor(shared(), G.METERS[_k]) >> monitor(shared(), G.METERS[(_k + 1) % 3])
                                                       >> lowpass_hz(1050.0, 1.0)) | timer(shared()))


@pytest.mark.parametrize("name", sorted(EMUL))
def test_templates_on_host_emulation(name, tmp_path):
    from test_device_emul_cpu import emulate, oracle
    n = 64 * 30 + 37
    s = shared(700.0 if "cutoff" in name else 0.6)
    if "rate" in name or "timer_alone" in name:   # (host emulation and oracle at another rate too)
        want = oracle(EMUL[name](s), n, sr=44100.0)
        got, _ = emulate(EMUL[name](s), n, None, str(tmp_path), sr=44100.0)
        assert np.array_equal(got, want)
    want = oracle(EMUL[name](s), n)
    got, _ = emulate(EMUL[name](s), n, None, str(tmp_path))
    assert np.abs(want).max() > 1e-3
    assert np.array_equal(got, want), (name, int((got != want).sum()))


# ---- the GPU file on the CPU mock device
def test_gpu_shared_file_on_the_mock_device(mock_env):
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_shared.py"), "-m", "gpu", "-q",
                        "-p", "no:cacheprovider", "--tb=short"], capture_output=True, text=True, env=mock_env, cwd=ROOT, timeout=1800)
    tail = r.stdout[-3000:]
    assert r.returncode == 0 and " passed" in tail and "failed" not in tail, tail

"""`GpuBank.set_voices` (fdsp_bank_set_voices): one Setting kind and address applied to many (voice, values) entries in one call.
It must do exactly what a loop of `GpuBank.set` calls does. So every case drives twin banks: A takes the batch and B takes the same
entries one `set` at a time, in order. Their rows must be bit for bit equal after the batch, and again after reset, clone,
set_sample_rate, a grow, another batch and a per-voice set. The headline bank is also checked against oracle units that take the same
sets at the same call boundaries, and its mix against the summation-order model of tests/test_gpu_mix.py."""
import ctypes as C
import os

import numpy as np
import pytest

from fundsp_b200 import workloads
from fundsp_b200.capi import FdspError, ERR_ARG
from fundsp_b200.net import Net
from fundsp_b200.prelude import *  # noqa: F401,F403
from fundsp_b200.sequencer import event, slot

pytestmark = pytest.mark.gpu
SR = 48000.0
MOCK = "mock" in os.environ.get("FDSP_B200_LIB", "")
V = 24
(P_CENTER, P_CENTER_Q, P_CENTER_Q_GAIN, P_VALUE, P_COEFFICIENT, P_BIQUAD, P_DELAY, P_TIME, P_ROUGHNESS, P_VARIABILITY, P_PAN,
 P_ATTACK_RELEASE, P_PHASE, P_SEED, P_INTERVAL) = range(1, 16)
R = ((1, 1),)          # .right()


def fv(i, k=0):
    return ((i * 37 + k * 11) % 29) / 29.0


def saw_i(i):
    return saw_hz(110.0 + 7.0 * i)


def lp():
    return lowpass_hz(1000.0, 1.0)


# name: (voice i, kind, address, entry values (rng, n) -> [n, nvalues])
def _u(lo, hi, k=1):
    return lambda g, n: g.uniform(lo, hi, (n, k))


BQ = lambda g, n: np.stack([-1.8 + 0.1 * g.uniform(0, 1, n), 0.82 + 0.05 * g.uniform(0, 1, n), 0.005 + 0.0 * g.uniform(0, 1, n),
                            np.full(n, 0.01), np.full(n, 0.005)], axis=1)
CASES = {
    # every kind fdsp_bank_set takes, on a node that takes it
    "center": (lambda i: saw_i(i) >> lp(), P_CENTER, R, _u(200.0, 5000.0)),
    "center_q": (lambda i: saw_i(i) >> lp(), P_CENTER_Q, R, lambda g, n: np.stack([g.uniform(200, 5000, n), g.uniform(0.5, 8, n)], 1)),
    "center_q_gain": (lambda i: saw_i(i) >> bell_hz(1000.0, 1.0, 2.0), P_CENTER_Q_GAIN, R,
                      lambda g, n: np.stack([g.uniform(200, 5000, n), g.uniform(0.5, 8, n), g.uniform(0.25, 4, n)], 1)),
    "value_dc": (lambda i: (dc(110.0 + i) >> saw()) >> lp(), P_VALUE, ((1, 0), (1, 0)), _u(50.0, 900.0)),
    "coefficient_allnest": (lambda i: noise().seed(i) >> allnest_c(0.3, lp()), P_COEFFICIENT, R, _u(-0.9, 0.9)),
    "biquad": (lambda i: saw_i(i) >> biquad(-1.8, 0.82, 0.005, 0.01, 0.005), P_BIQUAD, R, BQ),
    "delay_allpole": (lambda i: noise().seed(i) >> allpole_delay(0.5 + fv(i)), P_DELAY, R, _u(0.1, 3.0)),
    "time_follow": (lambda i: saw_i(i) >> follow(0.01 + 0.001 * i), P_TIME, R, _u(0.001, 0.2)),
    "roughness_dsf": (lambda i: dc(220.0 + i) >> dsf_saw_r(0.5), P_ROUGHNESS, R, _u(0.0, 1.0)),
    "pan": (lambda i: saw_i(i) >> pan(0.0), P_PAN, R, _u(-1.0, 1.0)),
    "attack_release_afollow": (lambda i: saw_i(i) >> afollow(0.01, 0.1), P_ATTACK_RELEASE, R, _u(0.001, 0.3, 2)),
    "phase_sine": (lambda i: (dc(220.0 + i) >> sine()) >> lp(), P_PHASE, ((1, 0), (1, 1)), _u(0.0, 1.0)),
    "seed_noise": (lambda i: noise().seed(i) >> lp(), P_SEED, ((1, 0),), lambda g, n: np.zeros((n, 0))),
    "interval_adsr": (lambda i: sine_hz(30.0 + i) >> adsr_live(0.01, 0.02, 0.5, 0.05), P_INTERVAL, R, _u(0.001, 0.01)),
    # settings that reach a node that ignores them, or lead nowhere
    "variability_ignored": (lambda i: saw_i(i) >> lp(), P_VARIABILITY, R, _u(0.0, 1.0)),
    "center_on_the_oscillator": (lambda i: saw_i(i) >> lp(), P_CENTER, ((1, 0), (1, 1)), _u(200.0, 5000.0)),
    "address_leads_nowhere": (lambda i: saw_i(i) >> lp(), P_CENTER, ((1, 7),), _u(200.0, 5000.0)),
    # addresses through every combinator a setting walks
    "stack": (lambda i: (saw_i(i) >> lp()) | (saw_i(i + 1) >> highpass_hz(500.0, 1.0)), P_CENTER, ((1, 1), (1, 1)), _u(200.0, 5000.0)),
    "branch": (lambda i: saw_i(i) >> (lp() ^ highpass_hz(500.0, 1.0)), P_CENTER_Q, ((1, 1), (1, 0)),
               lambda g, n: np.stack([g.uniform(200, 5000, n), g.uniform(0.5, 8, n)], 1)),
    "bus": (lambda i: saw_i(i) >> (lp() & bandpass_hz(1500.0, 2.0)), P_CENTER, ((1, 1), (1, 1)), _u(200.0, 5000.0)),
    "binop": (lambda i: (saw_i(i) >> lp()) + (saw_i(i + 3) >> highpass_hz(800.0, 1.0)), P_CENTER, ((1, 0), (1, 1)), _u(200.0, 5000.0)),
    "unop": (lambda i: saw_i(i) >> (lp() * 0.5), P_CENTER, R, _u(200.0, 5000.0)),
    "thru": (lambda i: saw_i(i) >> thru(lp()), P_CENTER, R, _u(200.0, 5000.0)),
    "multi": (lambda i: saw_i(i) >> split(3) >> stacki(3, lambda k: lowpass_hz(600.0 + 300.0 * k, 1.0)), P_CENTER, ((1, 1), (1, 2)),
              _u(200.0, 5000.0)),
    # entries that take the per-voice path
    "slot": (lambda i: slot(saw_i(i) >> lp()), P_CENTER, R, _u(200.0, 5000.0)),
    "update": (lambda i: update(saw_i(i) >> lp() >> highpass_hz(100.0, 1.0), 0.004,
                                "|t, dt, x| x.set(Setting::center(600.0 + 400.0 * sin_hz(r, t)).left().right())", r=1.0 + fv(i)),
               P_CENTER, ((1, 0), (1, 1)), _u(200.0, 5000.0)),
    "update_elsewhere": (lambda i: update(saw_i(i) >> lp() >> highpass_hz(100.0, 1.0), 0.004,
                                          "|t, dt, x| x.set(Setting::center(600.0 + 400.0 * sin_hz(r, t)).left().right())", r=1.0 + fv(i)),
                         P_CENTER, R, _u(50.0, 500.0)),
}


def pair(voices, **kw):
    from fundsp_b200.bank import GpuBank
    return GpuBank(voices(), sample_rate=SR, per_voice=True, **kw), GpuBank(voices(), sample_rate=SR, per_voice=True, **kw)


def entries(rng, nvoices, n, values):
    vs = rng.integers(0, nvoices, n).astype(np.uint32)
    vs[: min(n, nvoices)] = rng.permutation(nvoices)[:n]   # every voice, then duplicates (the last one wins)
    return vs, np.asarray(values(rng, n), np.float32)


def both(a, b, kind, vals, voices=None, seeds=None, address=()):
    """The batch on A, the loop on B."""
    a.set_voices(kind, vals, voices=voices, seeds=seeds, address=address)
    for j in range(vals.shape[0]):
        b.set(j if voices is None else int(voices[j]), kind, tuple(float(x) for x in vals[j]), seed=0 if seeds is None else int(seeds[j]),
              address=address)


def same(a, b, n, what):
    ga, gb = a.render_samples(n)[0], b.render_samples(n)[0]
    assert ga.shape == gb.shape and np.isfinite(ga).all(), what
    bad = int((ga != gb).sum())
    assert bad == 0, (what, bad)
    return ga


def twin_run(a, b, batch, grow=None, n=700):
    """The batch, then every operation after which A and B must still agree; `batch(a, b, rng)` applies one batch to both."""
    rng = np.random.default_rng(3)
    same(a, b, 300, "before")
    batch(a, b, rng)
    g = same(a, b, n, "after the batch")
    batch(a, b, rng)
    same(a, b, 64 * 3 + 5, "after a second batch")
    a.reset(); b.reset()
    same(a, b, n, "after reset")
    ca, cb = a.clone(), b.clone()
    same(ca, cb, n, "clones")
    a.set_sample_rate(44100.0); b.set_sample_rate(44100.0)
    same(a, b, n, "after set_sample_rate")
    if grow:
        grow(a); grow(b)
        same(a, b, 333, "after the bank grew")
        batch(a, b, rng)
        same(a, b, 333, "after a batch on the grown bank")
    return g


@pytest.mark.parametrize("name", sorted(CASES))
def test_batch_equals_the_loop(name):
    mk, kind, addr, values = CASES[name]
    a, b = pair(lambda: [mk(i) for i in range(V)])

    def batch(a, b, rng):
        vs, vals = entries(rng, a.voices(), 2 * V + 5, values)
        seeds = rng.integers(0, 2 ** 63, len(vs), dtype=np.uint64) if kind == P_SEED else None
        both(a, b, kind, vals, vs, seeds, addr)

    g = twin_run(a, b, batch, grow=lambda x: x.add_voice(mk(V + 1)))
    assert np.abs(g).max() > 1e-4
    # a per-voice set after all of it
    vs, vals = entries(np.random.default_rng(9), 1, 1, values)
    seeds = [12345] if kind == P_SEED else None
    a.set(0, kind, tuple(float(x) for x in vals[0]), seed=seeds[0] if seeds else 0, address=addr)
    b.set(0, kind, tuple(float(x) for x in vals[0]), seed=seeds[0] if seeds else 0, address=addr)
    same(a, b, 200, "after a per-voice set")


MIXED = [lambda i: saw_i(i) >> lp(), lambda i: noise().seed(i) >> lp(), lambda i: (dc(110.0 + i) >> sine()) >> lp()]


def test_classes_interleaved_one_launch_per_class():
    kinds = [(i * 7) % 3 for i in range(3 * V)]
    a, b = pair(lambda: [MIXED[k](i) for i, k in enumerate(kinds)])
    assert len(a.classes()) == 3
    same(a, b, 200, "before")
    rng = np.random.default_rng(5)
    for n, touched in [(1, 1), (2, None), (64, 3), (3 * V, 3), (5 * V, 3)]:
        vs, vals = entries(rng, 3 * V, n, _u(200.0, 5000.0))
        l0 = a.launch_count()
        a.set_voices(P_CENTER, vals, voices=vs, address=R)
        want = len({kinds[v] for v in vs}) if touched is None else touched
        assert a.launch_count() - l0 == want, (n, a.launch_count() - l0, want)
        for j in range(n):
            b.set(int(vs[j]), P_CENTER, (float(vals[j, 0]),), address=R)
        same(a, b, 129, ("after", n))
    # voices=None: entry j is voice j; an empty batch changes nothing and launches nothing
    vals = np.linspace(300.0, 3000.0, 3 * V, dtype=np.float32)
    both(a, b, P_CENTER, vals.reshape(-1, 1), None, None, R)
    same(a, b, 200, "voices=None")
    l0 = a.launch_count()
    a.set_voices(P_CENTER, np.zeros((0, 1), np.float32), address=R)
    assert a.launch_count() == l0
    same(a, b, 200, "empty batch")


# what the device is given by one call, read from a CUDA trace (torch.profiler, in a process of its own so that torch's libraries stay out
# of the test process): per call one host-to-device copy and one scatter kernel per class touched, for any n
TRACE = '''
import sys, numpy as np
from torch.profiler import ProfilerActivity, profile
from fundsp_b200.bank import GpuBank
from fundsp_b200.prelude import lowpass_hz, noise, saw_hz
mk = [lambda i: saw_hz(110.0 + 7.0 * i) >> lowpass_hz(1000.0, 1.0), lambda i: noise().seed(i) >> lowpass_hz(1000.0, 1.0)]
V = 2000
b = GpuBank([mk[i % 2](i) for i in range(V)], per_voice=False, mix=True, sample_rate=48000.0)
b.render_samples(256)
for n in (1, 64, 1999, V, 3 * V):
    vs = (np.arange(n) * 7 % V).astype(np.uint32)
    b.set_voices(1, np.full((n, 1), 500.0, np.float32), voices=vs, address=((1, 1),))   # (staging grown outside the trace)
    b.render_samples(64)
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        b.set_voices(1, np.linspace(300.0, 3000.0, n, dtype=np.float32).reshape(-1, 1), voices=vs, address=((1, 1),))
        b.L.fdsp_bank_sync(b.h)
    keys = [(e.key, e.count) for e in p.key_averages()]
    h2d = sum(c for k, c in keys if k.startswith("Memcpy HtoD"))
    scat = sum(c for k, c in keys if "set_columns_kernel" in k)
    print("call", n, h2d, scat, len({int(v) % 2 for v in vs}), flush=True)
'''


def test_one_copy_and_one_scatter_per_class_in_the_trace():
    if MOCK:
        pytest.skip("a CUDA trace needs the GPU (the launch counts are checked above on the mock device too)")
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", TRACE], capture_output=True, text=True, cwd=root, timeout=600,
                       env=dict(os.environ, PYTHONPATH=root))
    calls = [ln.split()[1:] for ln in r.stdout.splitlines() if ln.startswith("call ")]
    assert r.returncode == 0 and len(calls) == 5, (r.stdout[-1500:], r.stderr[-1500:])
    for n, h2d, scat, classes in calls:
        assert int(h2d) == 1 and int(scat) == int(classes), (n, h2d, scat, classes)


def test_words_a_setting_does_not_touch_take_no_launch():
    """Phase and seed settings change reset-image words only: the batch writes no parameter word (and the loop's result is the same)."""
    a, b = pair(lambda: [(dc(220.0 + i) >> sine()) >> lp() for i in range(V)])
    same(a, b, 100, "before")
    l0 = a.launch_count()
    both(a, b, P_PHASE, np.linspace(0, 1, V, dtype=np.float32).reshape(-1, 1), None, None, ((1, 0), (1, 1)))
    assert a.launch_count() == l0
    same(a, b, 100, "running phase unchanged")
    a.reset(); b.reset()
    same(a, b, 300, "after reset: the new phases")


def test_net_bank_by_vertex():
    mk = lambda i: noise().seed(i) >> lowpass_hz(300.0 + 100.0 * i, 1.0) >> pan(0.0)

    def net():
        n = Net.wrap(mk(0))
        for i in range(1, V):
            n = n & Net.wrap(mk(i))
        return n
    from fundsp_b200.bank import GpuBank
    a, b = GpuBank.from_net(net(), per_voice=True, sample_rate=SR), GpuBank.from_net(net(), per_voice=True, sample_rate=SR)
    ids = [0] + [1 + 3 * (i - 1) for i in range(1, V)]
    voices = np.array([a.voice_of_vertex(x) for x in ids[::-1]], np.uint32)
    rng = np.random.default_rng(2)

    def batch(a, b, rng):
        vals = np.stack([rng.uniform(300, 4000, V), rng.uniform(0.5, 6, V)], 1).astype(np.float32)
        both(a, b, P_CENTER_Q, vals, voices, None, ((1, 0), (1, 1)))
        both(a, b, P_PAN, rng.uniform(-1, 1, (V, 1)).astype(np.float32), voices, None, R)
    twin_run(a, b, batch)
    # a crossfading vertex takes the per-voice path, the others the batch
    a.crossfade_voice(2, 1, 0.01, mk(40)); b.crossfade_voice(2, 1, 0.01, mk(40))
    same(a, b, 100, "crossfade started")
    batch(a, b, rng)
    same(a, b, 1000, "batch during the crossfade")
    batch(a, b, rng)
    same(a, b, 300, "batch after the crossfade")


def test_sequencer_events_running_and_finished():
    mk = lambda i: event(saw_i(i) >> lp(), (30.0 + 97.3 * i) / SR, (30.0 + 97.3 * i + (400.0 if i % 3 == 0 else 9000.0)) / SR, i % 2,
                         40.0 / SR, 100.0 / SR)
    a, b = pair(lambda: [mk(i) for i in range(V)], mix=True)

    def batch(a, b, rng):
        vs, vals = entries(rng, a.voices(), V + 7, _u(200.0, 5000.0))
        both(a, b, P_CENTER, vals, vs, None, R)
    twin_run(a, b, batch, grow=lambda x: x.push_event(mk(V + 3)))


def test_refusal_mid_batch():
    """The first entry the loop would refuse: same error, same index; the entries before it applied, the rest not."""
    a, b = pair(lambda: [saw_i(i) >> lp() for i in range(V)])
    same(a, b, 100, "before")
    vs = np.array([3, 5, 3, 7, V + 2, 1, 2], np.uint32)
    vals = np.linspace(300.0, 2000.0, len(vs), dtype=np.float32).reshape(-1, 1)
    with pytest.raises(FdspError) as e:
        a.set_voices(P_CENTER, vals, voices=vs, address=R)
    assert e.value.code == ERR_ARG and e.value.entry == 4
    for j in range(4):
        b.set(int(vs[j]), P_CENTER, (float(vals[j, 0]),), address=R)
    with pytest.raises(FdspError) as e2:
        b.set(int(vs[4]), P_CENTER, (float(vals[4, 0]),), address=R)
    assert str(e2.value) == str(e.value)
    same(a, b, 500, "after the refusal")


# ---- the headline bank: every voice's cutoff and q, and its frequency dc, before every call
def test_headline_bank_against_oracle_units(monkeypatch):
    from fundsp_b200.bank import GpuBank
    from oracle import OracleUnit, lib as olib
    from test_gpu_mix import bank_classes, check_mix, launch_segments
    olib().fo_set_denormal_emulation(0)
    nv = 300 if MOCK else 16384
    voices = lambda: [workloads.saw_svf_voice(i) for i in range(nv)]   # noqa: E731
    calls = [64, 1000, 7, 61, 1000, 64, 1, 33, 1000, 64, 17]
    outs = {}
    for rt in ("1", "0"):
        monkeypatch.setenv("FDSP_RT", rt)
        bm, bv = GpuBank(voices(), per_voice=False, mix=True, sample_rate=SR), GpuBank(voices(), per_voice=True, sample_rate=SR)
        classes = bank_classes(bv, voices())
        rng = np.random.default_rng(17)
        got = []
        for k, n in enumerate(calls):
            cq = np.stack([rng.uniform(200, 8000, nv), rng.uniform(0.5, 8, nv)], 1).astype(np.float32)
            f = rng.uniform(55, 1760, (nv, 1)).astype(np.float32)
            for bank in (bm, bv):
                bank.set_voices(P_CENTER_Q, cq, address=R)
                bank.set_voices(P_VALUE, f, voices=np.arange(nv, dtype=np.uint32)[::-1].copy(), address=((1, 0), (1, 0)))
                # (entry j is voice V-1-j: the values in reverse order)
            if n > 64:
                rows, _ = bv.render_samples(n)
                _, mix = bm.render_samples(n)
                segs = launch_segments(n, classes, nv, 1, False, False)
            else:
                rows = bv.process(n).reshape(nv, 1, n)
                mix = bm.process(n)
                segs = [(0, n)]
            check_mix(mix, rows, classes, segs, False, (rt, k, n))
            got.append((rows, mix, cq, f))
        outs[rt] = got
    for (r1, m1, _, _), (r0, m0, _, _) in zip(outs["1"], outs["0"]):
        assert np.array_equal(r1, r0) and np.array_equal(m1, m0), "FDSP_RT=1 and FDSP_RT=0 differ"
    # oracle units with the same sets at the same call boundaries (a sample of voices on the GPU: every voice's rows are tied to the
    # mix model above, and the set path is the same for every voice of the class)
    pick = range(nv) if MOCK else sorted(set(range(0, nv, 97)) | {nv - 1})
    for v in pick:
        u = OracleUnit(workloads.saw_svf_voice(v)); u.set_sample_rate(SR)
        for (rows, _, cq, f), n in zip(outs["1"], calls):
            u.L.fo_set(u.h, P_CENTER_Q, (C.c_float * 2)(*cq[v]), 2, 0, (C.c_int64 * 2)(1, 1), 1)
            u.L.fo_set(u.h, P_VALUE, (C.c_float * 1)(f[nv - 1 - v, 0]), 1, 0, (C.c_int64 * 4)(1, 0, 1, 0), 2)
            want = u.process_many(n) if n > 64 else u.process(n)
            assert np.array_equal(rows[v], want.reshape(rows[v].shape)), (v, n, int((rows[v] != want.reshape(rows[v].shape)).sum()))
